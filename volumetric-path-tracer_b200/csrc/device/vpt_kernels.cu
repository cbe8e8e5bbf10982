// vpt_kernels.cu -- sm_90a wavefront kernels that replace the reference megakernel
// `volume_rt_kernel` (source/render_kernel.cu:2216-2326), both integrators.
//
//   k_prepare_scene : GPU_VDB[] + OCTNode tree (the reference launch parameters) -> flat scene tables
//   k_bn_prepare    : per-chunk blue-noise jitter table + golden-ratio advance of the 256x256 buffer (race-free, quirk Q6)
//   k_miss_cull     : once per render call of a pinhole frame: the pixels whose every jitter misses the root box and the sphere
//   k_generate      : one block per 32x4 pixel tile, all passes of the chunk: Philox stream, jitter, thin-lens ray,
//                     root/sphere test, draw-free prefix of the first tracking walk; misses write a 16-byte sample
//                     record, the rest are pushed into a warp-compacted ray queue (one atomic per warp); culled pixels sample nothing
//   k_trace<I, L, R, C, G> : persistent; every lane owns R rays parked in shared memory (vpt_trace.cuh); I = integrator (0 direct,
//                     1 volumetric path: vpt_trace_vol.cuh), L = lean instantiation for the common scene, C = cell table, G = light groups
//                     (the generic kernels also keep each ray's per-class radiance sums); k_trace_brick in brick mode.  The nine
//                     instantiations the host picks from (TraceKernel) are listed once, in trace_kernel below.
//   k_resolve<S, A, G> : per pixel, passes in order: environment term (S = 0 HDRI: with compact records for misses only; 1 / 2 precomputed
//                     sky: vpt_atmosphere.cuh), NaN guard, running mean, ACES tonemap, display/raw/depth/cost writes (the tail of the reference
//                     kernel); A: plus the running means of the compositing AOVs (alpha, volume colour), G: of the light groups (sun, point,
//                     emission, environment).  Its twelve instantiations, and those of k_resolve_adaptive, are listed in resolve_kernels below.
//   k_bn_advance, k_unpermute : blue-noise advance for non-sampling passes; stripe un-permutation after the multi-GPU gather
//   k_generate_adaptive, k_resolve_adaptive<S, A, G>, k_adapt : adaptive frames (vpt_render_adaptive) -- the same per-pixel work over the tiles
//                     that still hold an active pixel, a Welford state of the sample luminance, and the 3x3 convergence test;
//                     k_debug_adapt_pass feeds the same Welford state from caller-given samples (vpt_debug_adapt_rule)
//   k_adapt_halo, k_adapt_count_publish, k_adapt_tally, k_adapt_publish : the same frame sharded over the peer-memory exchange -- stripe-edge
//                     errors, the agreement on when to stop, and the final full-frame stores
//   k_layers_publish : depth, the compositing AOVs and the light groups into every rank's full-frame planes (vpt_comm_p2p_export_layers)
//   k_binned_publish : the deep slices or the instance mattes into every rank's full-frame [K][H][W] arrays (vpt_comm_p2p_export_binned)
//   k_generate_region, k_miss_cull_region, k_resolve_region<S, A, G>, k_adapt_init_region, k_adapt_region : render regions
//                     (vpt_set_render_region) -- the same per-pixel work over the pixels of one rectangle of the frame
//   k_generate_equirect, k_generate_adaptive_equirect, k_generate_region_equirect, k_miss_cull_equirect, k_miss_cull_region_equirect,
//   k_resolve_equirect<A, G>, k_resolve_adaptive_equirect<A, G>, k_resolve_region_equirect<A, G> : the equirectangular projection
//                     (vpt_set_projection) -- the same kernels with the camera ray of pano_b0; k_camera_rays: vpt_debug_camera_rays
//   k_generate_motion, k_generate_adaptive_motion, k_generate_region_motion : camera motion (vpt_set_camera_motion) -- k_generate with each
//                     sample's camera placed between two poses by its shutter draw (motion_camera); k_motion_cameras: vpt_debug_motion_cameras
//   k_generate_ods, k_generate_adaptive_ods, k_generate_region_ods : omni-directional stereo (vpt_set_projection_ods) -- k_generate with each
//                     sample's camera on its eye's viewing circle (ods_camera); k_ods_cameras: vpt_debug_ods_cameras, and the ODS camera rays
//   k_motion_vectors, k_motion_vectors_region, k_motion_vectors_adaptive (and their _motion forms) : motion vectors (vpt_set_motion_vectors)
//                     -- each sample's first collision projected through the frame camera and a second pose, next to the frame's resolve
//   k_collision_aovs, k_collision_aovs_region, k_collision_aovs_adaptive (and their _motion forms) : collision AOVs (vpt_set_collision_aovs)
//                     -- the world position, density normal and albedo at each sample's first collision, next to the frame's resolve
//   k_cryptomatte, k_cryptomatte_region, k_cryptomatte_adaptive : the Cryptomatte (vpt_set_cryptomatte) -- each pixel's collided samples
//                     counted by instance id, next to the frame's resolve; k_cryptomatte_rank : its ranks (vpt_cryptomatte_rank)
//
// Numerics: compiled with the reference's flags (--use_fast_math); decision-relevant expressions keep the reference
// build's operation order (read off its SASS) so a pixel's path is reproduced sample for sample (see vpt_math.cuh).
#include "vpt_frame.cuh"
#include "vpt_film.cuh"

namespace vpt {

// =====================================================================================================
// k_prepare_scene
// =====================================================================================================
// root == nullptr: the octree was built by vpt_octree_build, its flat tables already exist (`hdr` names them, any number of
// instances) and only the per-volume records -- which depend on the GPU_VDB[] array handed in at render time -- are made here.
// One kernel for both cases on purpose: the record arithmetic is then the very same machine code.
__global__ void k_prepare_scene(const vpt_gpu_vdb* __restrict__ vols, const vpt_octnode* __restrict__ root,
                                SceneTables* out, OctInternal* internal, uint2* leaf_list, int* leaf_indices,
                                VolumeRec* vrec, int max_volumes, const SceneTables hdr)
{
    const int tid = blockIdx.x * blockDim.x + threadIdx.x;
    const int nthreads = gridDim.x * blockDim.x;
    const int N = root ? root->num_volumes : hdr.num_volumes;
    if (!root && tid == 0) { SceneTables t = hdr; t.volumes = vrec; *out = t; }

    if (root && tid == 0) {
        out->root_pmin[0] = root->bbox.pmin.x; out->root_pmin[1] = root->bbox.pmin.y; out->root_pmin[2] = root->bbox.pmin.z;
        out->root_pmax[0] = root->bbox.pmax.x; out->root_pmax[1] = root->bbox.pmax.y; out->root_pmax[2] = root->bbox.pmax.z;
        out->max_extinction = root->max_extinction;
        out->min_extinction = root->min_extinction;
        out->num_volumes = N;
        out->single_volume = (N == 1) ? 1 : 0;
        out->internal = internal; out->leaf_list = leaf_list; out->leaf_indices = leaf_indices; out->volumes = vrec;
        out->leaf_nodes = nullptr;
    }

    // internal nodes: 0 = root, 1..8 = level 1, 9..72 = level 2
    for (int j = tid; root && j < kOctInternalNodes; j += nthreads) {
        const vpt_octnode* n = root;
        bool exists = true;
        if (j >= 1 && j < 9) { n = oct_ptr(root->children[j - 1]); }
        else if (j >= 9) {
            const int c1 = (j - 9) >> 3, c2 = (j - 9) & 7;
            const vpt_octnode* p = oct_ptr(root->children[c1]);
            if (p->num_volumes > 0) n = oct_ptr(p->children[c2]); else exists = false;
        }
        OctInternal o;
        for (int a = 0; a < 3; ++a) { o.pmin[a] = 0.f; o.half[a] = 0.f; o.pmax[a] = 0.f; }
        o.child_empty = 0xffu; o.pad[0] = o.pad[1] = 0u;
        if (exists && n->num_volumes > 0) {
            o.pmin[0] = n->bbox.pmin.x; o.pmin[1] = n->bbox.pmin.y; o.pmin[2] = n->bbox.pmin.z;
            o.pmax[0] = n->bbox.pmax.x; o.pmax[1] = n->bbox.pmax.y; o.pmax[2] = n->bbox.pmax.z;
            const vpt_octnode* c0 = oct_ptr(n->children[0]);       // child 0 = (x-, y+, z-)
            o.half[0] = c0->bbox.pmax.x; o.half[1] = c0->bbox.pmin.y; o.half[2] = c0->bbox.pmax.z;
            uint32_t mask = 0;
            for (int c = 0; c < 8; ++c) if (oct_ptr(n->children[c])->num_volumes == 0) mask |= 1u << c;
            o.child_empty = mask;
        }
        internal[j] = o;
    }

    // leaves: volume lists (instanced scenes); stride VPT_OCT_MAX_VOLUMES per leaf
    for (int l = tid; root && l < kOctLeaves; l += nthreads) {
        const int c1 = l >> 6, c2 = (l >> 3) & 7, c3 = l & 7;
        uint2 lst = make_uint2((uint32_t)l * VPT_OCT_MAX_VOLUMES, 0u);
        const vpt_octnode* p1 = oct_ptr(root->children[c1]);
        if (p1->num_volumes > 0) {
            const vpt_octnode* p2 = oct_ptr(p1->children[c2]);
            if (p2->num_volumes > 0) {
                const vpt_octnode* p3 = oct_ptr(p2->children[c3]);
                const int cnt = p3->num_volumes;
                lst.y = (uint32_t)cnt;
                if (N > 1) for (int i = 0; i < cnt; ++i) leaf_indices[lst.x + i] = p3->vol_indices[i];
            }
        }
        leaf_list[l] = lst;
    }

    // per-volume world->index affine
    for (int v = tid; v < N && v < max_volumes; v += nthreads) vrec[v] = make_volume_rec(vols[v]);
}

// =====================================================================================================
// k_generate
// =====================================================================================================
// kAdaptive: the grid runs over the active tiles of `ad` instead of all tiles, and a lane whose pixel has stopped samples nothing (no
// plane record, no ray).  Two kernels (k_generate, k_generate_adaptive) so the fixed-count one is the very same machine code as before.
// kRegion (k_generate_region): the grid runs over the tile rectangle of `rg`, and a lane whose pixel lies outside R samples nothing.
// kPano (k_generate_equirect, ...): the ray is (camera origin, normalize(pano_b0)) under the projection `pj` (lens_radius is 0, the host
// refuses anything else), and takes the pinhole branch below: its lens draws are counted after the box / octree prefix, as a pinhole's.
// kMotion (k_generate_motion, ...): the camera moves over the shutter (`mo`, the pose at shutter close).  The ray depends on the shutter
// draw, whose index depends on how many trials the lens loop took, so every sample runs the loop first, takes xi where the static kernels
// skip the shutter draw, and builds its ray from motion_camera(xi) in the thin-lens order (a pinhole's rd is +-0).  No pre-step: queue_aux
// carries the per-ray origin (the host sets thin_lens), and the host runs no miss cull.
// kOds (k_generate_ods, ...): each sample's camera is ods_camera's under `od` (its own origin, horizontal = vertical = 0), traced by the
// perspective rule below as the reference camera it is.  No pre-step and no miss cull, as for motion: queue_aux carries the origin.
template <bool kAdaptive, bool kRegion = false, bool kPano = false, bool kMotion = false, bool kOds = false>
__device__ __forceinline__ void generate_body(const FrameArgs& fa, const AdaptArgs* ad, const RenderRegion* rg = nullptr, const Projection* pj = nullptr,
                                              const CameraMotion* mo = nullptr, const OdsParams* od = nullptr)
{
    const FrameGeom& g = fa.geom;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int tiles_x = (g.width + 31) / 32;
    const int n_tiles = kAdaptive ? ad->n_tiles : kRegion ? (rg->tx1 - rg->tx0) * (rg->ty1 - rg->ty0) : tiles_x * ((g.local_rows + 3) / 4);
    // the tile of list entry ti: the active-tile list, R's tile rectangle row by row, or every tile
    auto tile_of = [&](const int ti) {
        if constexpr (kAdaptive) return (int)__ldg(ad->tiles + ti);
        else if constexpr (kRegion) { const int w = rg->tx1 - rg->tx0, r = ti / w; return (rg->ty0 + r) * tiles_x + rg->tx0 + (ti - r * w); }
        else return ti;
    };
    // a pixel of R (local row lr, column x)
    auto in_region = [&](const int x, const int lr) { return !kRegion || (x >= rg->x0 && x < rg->x1 && lr >= rg->lr0 && lr < rg->lr1); };
    // pixels culled by k_miss_cull (every jitter misses the box and the sphere) sample nothing here: k_resolve rebuilds their miss samples.
    // A block none of whose pixels samples leaves before staging anything; the vote is block-wide, so all its threads leave together.
    // (Every tile of R's rectangle holds a pixel of R, so without the cull a region block always has work.)
    if (fa.miss_mask) {
        bool idle = true;
        for (int ti = blockIdx.x * fa.tiles_per_block; ti < min(n_tiles, (int)(blockIdx.x + 1) * fa.tiles_per_block); ++ti) {
            const int tile = tile_of(ti);
            const int tile_y = tile / tiles_x;
            const int x = (tile - tile_y * tiles_x) * 32 + warp * 8 + (lane & 7), lr = tile_y * 4 + (lane >> 3);
            if (x < g.width && lr < g.local_rows && global_row(g, lr) < g.height && in_region(x, lr)) {
                const size_t lp = (size_t)lr * g.width + x;
                bool stopped = false;
                if constexpr (kAdaptive) stopped = ad->stopped[lp];
                if (!stopped && !fa.miss_mask[lp]) idle = false;
            }
        }
        if (__syncthreads_and(idle)) return;
    }

    __shared__ FrameShared fs;
    __shared__ float vdc2[101], vdc3[101];                     // radical inverses of 0..100 in bases 2 and 3
    // the lens sampler only ever asks for vanDerCorput(int(xi * 100)): tabulate it with the reference's own loop -- radical_inverse
    // (vpt_frame.cuh) written out, because calling it here moves the machine code of k_generate_adaptive
    if (threadIdx.x < 101) {
        { int n = threadIdx.x; float r = 0, denom = 1, inv = 1.f / 2; while (n) { denom *= 2; r = padd(r, __fdividef((float)(n % 2), denom)); n *= inv; } vdc2[threadIdx.x] = r; }
        { int n = threadIdx.x; float r = 0, denom = 1, inv = 1.f / 3; while (n) { denom *= 3; r = padd(r, __fdividef((float)(n % 3), denom)); n *= inv; } vdc3[threadIdx.x] = r; }
    }
    __shared__ EmptyAhead ea;
    load_frame_shared(fs, fa.scene, (!kMotion && !kOds) ? &ea : nullptr);   // the pre-step's table (none under motion / ODS)
    const SceneTables& sc = fs.sc;
    uint32_t n_pre = 0, n_hop = 0, n_ahead = 0;                 // statistics of the pre-step: rays, hops, rays ended by "empty ahead"

    const SphereRec sph = load_sphere(fa.sphere);
    // one block = a run of 32x4 pixel tiles x a run of passes: enough (tile, pass) pairs per block to amortise the octree / table staging
    // above -- many passes of one tile when passes are fused, several tiles when the caller renders pass by pass; a small local frame
    // (multi-GPU shard, low resolution) splits the chunk's passes over blockIdx.z instead: see launch_generate
    for (int ti = blockIdx.x * fa.tiles_per_block; ti < min(n_tiles, (int)(blockIdx.x + 1) * fa.tiles_per_block); ++ti) {
    const int tile = tile_of(ti);
    const int tile_y = tile / tiles_x, tile_x = tile - tile_y * tiles_x;
    const int x = tile_x * 32 + warp * 8 + (lane & 7);
    const int lr = tile_y * 4 + (lane >> 3);
    const int y = global_row(g, lr);
    bool valid = (x < g.width) && (lr < g.local_rows) && (y < g.height);
    if constexpr (kAdaptive) { if (valid && ad->stopped[(size_t)lr * g.width + x]) valid = false; }
    if constexpr (kRegion) { if (!in_region(x, lr)) valid = false; }
    if (valid && fa.miss_mask && fa.miss_mask[(size_t)lr * g.width + x]) valid = false;

    const int pass_begin = blockIdx.z * fa.passes_per_block;
    const int pass_end = min(fa.n_passes, pass_begin + fa.passes_per_block);
    // blue-noise jitter of each pass, from the per-chunk table written by k_bn_prepare; the value of the NEXT pass is requested one
    // iteration ahead (the load was the kernel's top stall: every pass started by waiting ~1 us for these 8 bytes)
    const int bn_index = valid ? (y % 256) * 256 + (x % 256) : 0;
    float2 bn_next = (valid && pass_begin < pass_end) ? __ldg(fa.bn_table + (size_t)pass_begin * 65536 + bn_index) : make_float2(0.f, 0.f);
    for (int pass = pass_begin; pass < pass_end; ++pass) {
    const float2 bnv = bn_next;
    if (valid && pass + 1 < pass_end) bn_next = __ldg(fa.bn_table + (size_t)(pass + 1) * 65536 + bn_index);
    bool hit = false;
    float3 org = f3(0.f), dir = f3(0.f, 0.f, 1.f);
    uint32_t kdraws = 0;
    int obj = 0; float t_min = 0.f;
    bool prestepped = false; float3 wstart = f3(0.f);
    const uint32_t lp = (uint32_t)lr * (uint32_t)g.width + (uint32_t)x;

    if (valid) {
        const vpt_kernel_params& kp = fa.kp;
        const vpt_camera& cam = fa.cam;
        const uint32_t idx = (uint32_t)y * (uint32_t)g.width + (uint32_t)x;
        Rng rng; rng.init(idx, kp.iteration + (uint32_t)pass, 0u);

        // thin-lens ray (reference camera::get_ray, camera.h:131-136).  The lens sample is drawn by a rejection loop on the pixel's
        // Philox stream BEFORE the ray exists -- but with a pinhole (lens_radius == 0) the sample is multiplied by zero: the ray
        // does not depend on it and the only thing the path needs from the loop is HOW MANY draws it consumed.  So the pinhole ray is
        // built first, the box / octree prefix below decides whether the sample can hit anything, and only the survivors run the
        // generator (70 % of the samples of the headline frame are misses and never touch it).  Bit-exactness: offset = u*0*p.x +
        // v*0*p.y is +-0; x + (+-0) == x and x - (+-0) == x for every x != 0, so lanes where a zero could meet a signed zero
        // (an origin or direction component that is exactly 0) take the literal order instead.
        bool lens_pending = false;
        if constexpr (kPano) {
            // no lens offset is ever added, so no signed zero can meet the origin or b0: every sample takes the pinhole order
            org = ld3(cam.origin);
            dir = normalize(pano_b0(cam, *pj, kp.resolution, x, y, bnv.x, bnv.y));
            lens_pending = true;
        } else if constexpr (kMotion) {
            float3 p;
            do {
                const float a = vdc2[int(rng.next() * 100)];
                const float b = vdc3[int(rng.next() * 100)];
                p = f3(pfma(a, 2.0f, -1.0f), pfma(b, 2.0f, -1.0f), 0.0f);
            } while (pfma(p.x, p.x, pmul(p.y, p.y)) >= 1.0f);
            const vpt_camera mc = motion_camera(cam, *mo, rng.next());  // the shutter-time draw places the camera between the poses
            const float3 rd = f3(pmul(cam.lens_radius, p.x), pmul(cam.lens_radius, p.y), 0.0f);
            const float3 offset = f3(pfma(mc.u.x, rd.x, pmul(mc.v.x, rd.y)), pfma(mc.u.y, rd.x, pmul(mc.v.y, rd.y)), pfma(mc.u.z, rd.x, pmul(mc.v.z, rd.y)));
            const float3 b0 = camera_b0(mc, kp.resolution, x, y, bnv.x, bnv.y);
            org = f3(padd(mc.origin.x, offset.x), padd(mc.origin.y, offset.y), padd(mc.origin.z, offset.z));
            dir = normalize(f3(psub(b0.x, offset.x), psub(b0.y, offset.y), psub(b0.z, offset.z)));
            kdraws = rng.k;
        } else {
            vpt_camera ocam;
            if constexpr (kOds) ocam = ods_camera(cam, *od, kp.resolution, x, y, bnv.x, bnv.y).cam;
            const vpt_camera& pc = kOds ? ocam : cam;         // the camera whose ray the sample is
            const bool pinhole = pinhole_camera(pc);
            const float3 b0 = camera_b0(pc, kp.resolution, x, y, bnv.x, bnv.y);
            if (pinhole && b0.x != 0.0f && b0.y != 0.0f && b0.z != 0.0f) {
                org = ld3(pc.origin);
                dir = normalize(b0);
                lens_pending = true;
            } else {
                float3 p;
                do {
                    const float a = vdc2[int(rng.next() * 100)];
                    const float b = vdc3[int(rng.next() * 100)];
                    p = f3(pfma(a, 2.0f, -1.0f), pfma(b, 2.0f, -1.0f), 0.0f);
                } while (pfma(p.x, p.x, pmul(p.y, p.y)) >= 1.0f);
                const float3 rd = f3(pmul(pc.lens_radius, p.x), pmul(pc.lens_radius, p.y), 0.0f);
                const float3 offset = f3(pfma(pc.u.x, rd.x, pmul(pc.v.x, rd.y)), pfma(pc.u.y, rd.x, pmul(pc.v.y, rd.y)), pfma(pc.u.z, rd.x, pmul(pc.v.z, rd.y)));
                ++rng.k;                                                 // shutter time draw: consumed, value unused by the path
                org = f3(padd(pc.origin.x, offset.x), padd(pc.origin.y, offset.y), padd(pc.origin.z, offset.z));
                dir = normalize(f3(psub(b0.x, offset.x), psub(b0.y, offset.y), psub(b0.z, offset.z)));
                kdraws = rng.k;
            }
        }

        const bool sphere_clear = line_misses_sphere(sph, org, dir);   // then sphere::intersect is known to fail: skip it
        if (sphere_clear) { float tmax1; obj = aabb_intersect(sc.root_pmin, sc.root_pmax, org, dir, t_min, tmax1) ? 1 : 0; }
        else obj = closest_object(sc, sph, org, dir, t_min);
        hit = (obj != 0);

        // Draw-free prefix of the first delta walk: until the ray reaches a non-empty octree leaf the reference's `sample`
        // only hops over empty nodes (no random number is consumed).  Run those hops here, at full warp width; a ray that
        // leaves the box without ever meeting a populated leaf contributes exactly what a miss does and never enters the
        // queue, the others are queued at the position where stepping really starts.  (Pinhole camera and a ray whose line
        // provably misses the sphere only; everything else takes the generic route.)
        if (!kMotion && !kOds && obj == 1 && kp.ray_depth >= 1 && kp.volume_depth >= 1 && cam.lens_radius == 0.0f && sphere_clear) {
            float3 p = madd3(org, dir, padd(t_min, VPT_EPS));
            int leaf = -2;
            if (!aabb_contains(sc.root_pmin, sc.root_pmax, p)) leaf = -1;
            n_pre++;
            // -3: no populated leaf ahead, the hops would end outside the box -- the miss record needs only org and dir
            for (int it = 0; it < 256 && leaf == -2; ++it) { leaf = oct_locate_or_skip<true, true>(fs.oct, sc, p, dir, &ea); n_hop += (leaf == -2); }
            if (leaf == -3) { n_ahead++; leaf = -1; }
            if (leaf == -1) {                                    // walked out through empty space: sample == miss sample
                hit = false;
                if (kp.integrator != 0) dir = normalize(dir);    // vol_integrator renormalises after a box hit (:1747)
            }
            else if (leaf >= 0) { prestepped = true; wstart = p; }
            // leaf == -2 after 256 hops: leave it to the generic route
        }

        if (hit && lens_pending) {
            // the rejection loop, for its draw count only (2 per trial + the shutter-time draw)
            float px, py;
            do {
                px = pfma(vdc2[int(rng.next() * 100)], 2.0f, -1.0f);
                py = pfma(vdc3[int(rng.next() * 100)], 2.0f, -1.0f);
            } while (pfma(px, px, pmul(py, py)) >= 1.0f);
            kdraws = rng.k + 1u;
        }

        if (!hit) {
            const size_t s = (size_t)pass * g.n_local + lp;
            // 16-byte miss record: direction + sentinel (L = 0, beta = 1, depth = 0, tr = 0 are implied; planes B/C untouched)
            fa.planeA[s] = make_float4(dir.x, dir.y, dir.z, __uint_as_float(kMissSentinel));
            if (fa.planeD) fa.planeD[s] = make_float4(org.x, org.y, org.z, 0.f);
        }
    }

    // warp-compacted push: one atomic per warp, records contiguous per 8x4 pixel tile
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if (m) {
        unsigned base = 0;
        if (lane == __ffs(m) - 1) base = atomicAdd(fa.queue_count, __popc(m));
        base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
        if (hit) {
            // 24-byte record (+16 B origin when the lens is not a pinhole): direction + entry distance, ids + RNG position
            const unsigned slot = base + __popc(m & ((1u << lane) - 1u));
            fa.queue_dir[slot] = make_float4(dir.x, dir.y, dir.z, t_min);
            fa.queue_id[slot] = make_uint2(ray_pixel_word(g, lr, x), (uint32_t)pass | (kdraws << 6) | ((uint32_t)obj << 16) | ((uint32_t)prestepped << 18));
            if (prestepped) fa.queue_aux[slot] = make_float4(wstart.x, wstart.y, wstart.z, 0.f);      // where stepping starts
            else if (fa.thin_lens) fa.queue_aux[slot] = make_float4(org.x, org.y, org.z, 0.f);   // thin lens: per-ray origin
        }
    }
    }   // pass loop
    }   // tile loop

    if (fa.counters) {                                           // optional statistics: [12] pre-step rays, [13] hops, [14] ended at once
        for (int o = 16; o > 0; o >>= 1) {
            n_pre += __shfl_xor_sync(0xffffffffu, n_pre, o); n_hop += __shfl_xor_sync(0xffffffffu, n_hop, o); n_ahead += __shfl_xor_sync(0xffffffffu, n_ahead, o);
        }
        if (lane == 0) {
            atomicAdd(fa.counters + 12, (unsigned long long)n_pre); atomicAdd(fa.counters + 13, (unsigned long long)n_hop);
            atomicAdd(fa.counters + 14, (unsigned long long)n_ahead);
        }
    }
}

__global__ void __launch_bounds__(128)
k_generate(const FrameArgs fa) { generate_body<false>(fa, nullptr); }

__global__ void __launch_bounds__(128)
k_generate_adaptive(const FrameArgs fa, const AdaptArgs ad) { generate_body<true>(fa, &ad); }

__global__ void __launch_bounds__(128)
k_generate_region(const FrameArgs fa, const RenderRegion rg) { generate_body<false, true>(fa, nullptr, &rg); }

__global__ void __launch_bounds__(128)
k_generate_equirect(const FrameArgs fa, const Projection pj) { generate_body<false, false, true>(fa, nullptr, nullptr, &pj); }

__global__ void __launch_bounds__(128)
k_generate_adaptive_equirect(const FrameArgs fa, const AdaptArgs ad, const Projection pj) { generate_body<true, false, true>(fa, &ad, nullptr, &pj); }

__global__ void __launch_bounds__(128)
k_generate_region_equirect(const FrameArgs fa, const RenderRegion rg, const Projection pj) { generate_body<false, true, true>(fa, nullptr, &rg, &pj); }

__global__ void __launch_bounds__(128)
k_generate_motion(const FrameArgs fa, const CameraMotion mo) { generate_body<false, false, false, true>(fa, nullptr, nullptr, nullptr, &mo); }

__global__ void __launch_bounds__(128)
k_generate_adaptive_motion(const FrameArgs fa, const AdaptArgs ad, const CameraMotion mo) { generate_body<true, false, false, true>(fa, &ad, nullptr, nullptr, &mo); }

__global__ void __launch_bounds__(128)
k_generate_region_motion(const FrameArgs fa, const RenderRegion rg, const CameraMotion mo) { generate_body<false, true, false, true>(fa, nullptr, &rg, nullptr, &mo); }

__global__ void __launch_bounds__(128)
k_generate_ods(const FrameArgs fa, const OdsParams od) { generate_body<false, false, false, false, true>(fa, nullptr, nullptr, nullptr, nullptr, &od); }

__global__ void __launch_bounds__(128)
k_generate_adaptive_ods(const FrameArgs fa, const AdaptArgs ad, const OdsParams od)
{ generate_body<true, false, false, false, true>(fa, &ad, nullptr, nullptr, nullptr, &od); }

__global__ void __launch_bounds__(128)
k_generate_region_ods(const FrameArgs fa, const RenderRegion rg, const OdsParams od)
{ generate_body<false, true, false, false, true>(fa, nullptr, &rg, nullptr, nullptr, &od); }

// The render call's empty-ahead table, into the scene allocation (one CTA): the table depends only on the octree and the option, so it
// is built once here instead of by every block of k_generate and k_trace
__global__ void __launch_bounds__(128)
k_empty_ahead(SceneAlloc* scene, int enable)
{
    __shared__ FrameShared fs;
    __shared__ AheadScratch s;
    load_frame_shared(fs, &scene->sc);
    build_empty_ahead(scene->ahead, s, fs.oct, enable != 0);
}

// =====================================================================================================
// k_miss_cull
// =====================================================================================================
// One thread per strip of kCullStrip pixels of a local row, once per render call.  The strip's pixels are culled (mask 1) only when
//   (a) the camera is a pinhole (pinhole_camera);
//   (b) every component of b0 keeps one strict sign over the strip's closed jitter range (x + jx from x0 to x1, y + jy from y to y + 1),
//       away from 0 by kCullSignMargin of the largest: each operation of camera_b0 is monotone in x + jx and in y + jy, so every b0 of
//       the strip lies in the box D spanned by its values at the four corners, computed here by the same helper (the same bits).
//       k_generate then takes the pinhole branch for every sample;
//   (c) a plane through the camera origin has every root-box corner on one side and every d of D at least kCullSlack |d| inside the other
//       (candidates: the coordinate planes and the planes through two box corners, which include the facets of the cone over the box);
//   (d) the sphere, grown as in line_misses_sphere (r'^2 = 1.02 r^2 + 2e-3 |c - o|^2 + 1e-6), is further than kCullSlack from a circular
//       cone holding D.
// Then every ray of the pixel passes the box and the sphere at an angle of at least kCullSlack (1e-3 rad, about 8000 float ulps: far
// beyond the rounding of normalize and of the float slab and quadratic tests), so k_generate finds obj == 0 and stores direction +
// kMissSentinel -- what k_resolve rebuilds.  (c) and (d) are evaluated in double.  A pixel near a silhouette that is not culled only
// costs time.
constexpr double kCullSlack = 1e-3, kCullSignMargin = 1e-3, kCullPlaneTol = 1e-9;
constexpr int kCullPlanes = 6 + 2 * 28;
constexpr int kCullStrip = 4;                   // pixels of one row tested together (one box D for the strip)

__device__ __forceinline__ double3 box_corner(const double pmin[3], const double pmax[3], const int i, const double3 o)
{
    return make_double3(((i & 1) ? pmax[0] : pmin[0]) - o.x, ((i & 2) ? pmax[1] : pmin[1]) - o.y, ((i & 4) ? pmax[2] : pmin[2]) - o.z);
}
__device__ __forceinline__ double dot_d(const double3 a, const double3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ double len_d(const double3 a) { return sqrt(dot_d(a, a)); }
// ODS: the squared radius of the sphere grown as line_misses_sphere grows it for an origin up to R from the camera origin (distance <= L + R),
// then by R
__device__ __forceinline__ double ods_grown_r2(const float radius, const double L2, const double R)
{
    const double L = sqrt(L2) + R;
    const double rb = sqrt(1.02 * (double)radius * (double)radius + 2e-3 * L * L + 1e-6) + R;
    return rb * rb;
}

// The equirectangular strip x0 .. x1 - 1 of global row y (tests (a) - (d) of miss_cull_body, kPano).  The float angles of its samples lie in
// [phi(x0 + 0), phi(x1 + 0)] x [theta(y + 0), theta(y + 1)] (pano_angles is monotone), computed here by the same helper (the same bits).  In
// the orthonormal frame (u, v, -w) a direction of that range is within |theta - theta_c| of (phi_c, theta) along a meridian, and that one
// within cos(theta) |phi - phi_c| of (phi_c, theta_c) along a parallel: the cone around f = d(phi_c, theta_c) of half-angle
// alpha = dtheta / 2 + max cos(theta) dphi / 2 holds them all, at the poles and at the seam too.  The stored basis is orthonormal only up
// to float rounding: with every entry of M^T M - I (M = [u v w]) at most e, M's condition number k has k^2 <= (1 + 3e) / (1 - 3e), and M
// moves no angle by more than 2 asin((k - 1) / (k + 1)), which alpha takes in.  The float rounding of __sinf / __cosf, pano_b0 and normalize
// (about 1e-6 rad) is far below kCullSlack.
template <bool kOds = false>
__device__ __forceinline__ bool pano_strip_culled(const vpt_camera& cam, const Projection& pj, const vpt_u2 res, const int x0, const int x1,
                                                  const int y, const double3* planes, const int n_planes, const double3 sa, const double L2,
                                                  const double r2, const double ods_delta = 0.0)
{
    const double3 U = make_double3(cam.u.x, cam.u.y, cam.u.z), V = make_double3(cam.v.x, cam.v.y, cam.v.z), Wd = make_double3(cam.w.x, cam.w.y, cam.w.z);
    const double e = fmax(fmax(fmax(fabs(dot_d(U, U) - 1.0), fabs(dot_d(V, V) - 1.0)), fmax(fabs(dot_d(Wd, Wd) - 1.0), fabs(dot_d(U, V)))),
                          fmax(fabs(dot_d(U, Wd)), fabs(dot_d(V, Wd))));
    if (!(e < 1e-4)) return false;                                // (also a NaN basis)
    const double k = sqrt((1.0 + 3.0 * e) / (1.0 - 3.0 * e));
    const float2 lo = pano_angles(pj, res, x0, y, 0.0f, 0.0f), hi = pano_angles(pj, res, x1, y, 0.0f, 1.0f);
    const double p0 = lo.x, p1 = hi.x, t0 = lo.y, t1 = hi.y;
    const double pc = (p0 + p1) / 2, tc = (t0 + t1) / 2;
    const double cmax = (t0 <= 0.0 && t1 >= 0.0) ? 1.0 : fmax(cos(t0), cos(t1));
    double alpha = (t1 - t0) / 2 + cmax * (p1 - p0) / 2 + 2.0 * asin((k - 1.0) / (k + 1.0));
    if constexpr (kOds) alpha += ods_delta;
    if (!(alpha + kCullSlack < 1.5707963267948966)) return false;
    const double ct = cos(tc), st = sin(tc), sp = sin(pc), cp = cos(pc);
    double3 f = make_double3(ct * (sp * U.x - cp * Wd.x) + st * V.x, ct * (sp * U.y - cp * Wd.y) + st * V.y, ct * (sp * U.z - cp * Wd.z) + st * V.z);
    const double fl = len_d(f);
    f = make_double3(f.x / fl, f.y / fl, f.z / fl);
    // ODS: every component of every ray direction is away from 0 (a unit vector within alpha of f moves each component by at most alpha),
    // so k_generate_ods takes the pinhole order for every sample and k_resolve_ods rebuilds it as normalize(camera_b0)
    if constexpr (kOds) {
        const double m = alpha + kCullSlack;
        if (!(fabs(f.x) > m && fabs(f.y) > m && fabs(f.z) > m)) return false;
    }
    // (c)
    const double lim = -sin(alpha + kCullSlack);
    bool box_miss = false;
    for (int i = 0; i < n_planes && !box_miss; ++i) box_miss = dot_d(f, planes[i]) < lim;
    if (!box_miss) return false;
    // (d): the angle between f and the sphere's centre exceeds alpha + asin(r' / L) + kCullSlack (below pi: alpha < pi / 2)
    return dot_d(f, sa) / sqrt(L2) < cos(alpha + asin(sqrt(r2 / L2)) + kCullSlack);
}

// The ODS cull's bounds (k_miss_cull_ods), in double, or a negative R when the camera cannot be culled:
//   R, the radius of a ball around the camera origin that holds every origin' of the frame: |s| <= ipd/2, |r| <= sqrt((1 + 2e)(1 + 1e-5))
//     + sqrt(3) 2^-23 (the float basis' error e as in pano_strip_culled, __sinf / __cosf within 2.5e-6 of the unit circle, the rounding of
//     r's components), and the fma rounds each component of origin' by at most 2^-24 |origin'|;
//   delta, the angle between llc' - origin' and b0: llc' and the subtraction round each component by at most 2^-24 (|origin'| + |b0|)
//     and 2^-24 |llc' - origin'|, against |b0| >= 0.9.
// Every origin component must be further than R from 0, so that no origin' component is 0 and the pinhole order is taken.
struct OdsCullBounds { double R, delta; };
__device__ __forceinline__ OdsCullBounds ods_cull_bounds(const vpt_camera& cam, const OdsParams& od)
{
    const double3 U = make_double3(cam.u.x, cam.u.y, cam.u.z), V = make_double3(cam.v.x, cam.v.y, cam.v.z), Wd = make_double3(cam.w.x, cam.w.y, cam.w.z);
    const double e = fmax(fmax(fmax(fabs(dot_d(U, U) - 1.0), fabs(dot_d(V, V) - 1.0)), fmax(fabs(dot_d(Wd, Wd) - 1.0), fabs(dot_d(U, V)))),
                          fmax(fabs(dot_d(U, Wd)), fabs(dot_d(V, Wd))));
    OdsCullBounds b; b.R = -1.0; b.delta = 0.0;
    if (!(e < 1e-4)) return b;
    const double u24 = 5.9604644775390625e-8, s3 = 1.7320508075688772;
    const double rb = sqrt((1.0 + 2.0 * e) * (1.0 + 1e-5)) + s3 * 2.0 * u24;
    const double h = fabs((double)od.half_ipd);
    const double omax = fmax(fmax(fabs((double)cam.origin.x), fabs((double)cam.origin.y)), fabs((double)cam.origin.z));
    const double R = (h * rb + s3 * u24 * (omax + h * rb)) * (1.0 + 1e-12);
    const double omin = fmin(fmin(fabs((double)cam.origin.x), fabs((double)cam.origin.y)), fabs((double)cam.origin.z));
    const double err = s3 * 2.0 * u24 * (omax + R + 2.0);
    if (!(isfinite(R) && omin > R && err < 0.45)) return b;
    b.R = R; b.delta = asin(fmin(1.0, err / (0.9 - err)));
    return b;
}

// kRegion (k_miss_cull_region): only the strips that hold a pixel of R -- the same strips, on the same kCullStrip grid, as a full frame.
// kPano (k_miss_cull_equirect, k_miss_cull_region_equirect): the equirectangular projection `pj`, whose rays all start at the camera
// origin.  (a) and (b) become: the camera has no lens, and the strip's directions lie in a cone of half-angle alpha < pi / 2 - kCullSlack
// around the direction f of the centre of its (phi, theta) range (see below).  (c) holds when f . n < -sin(alpha + kCullSlack) for a
// candidate plane n: every direction of the cone is then more than kCullSlack past the plane.  (d) is the test above with that cone.
// kOds (k_miss_cull_ods, k_miss_cull_region_ods): the ODS projection `od`.  Every origin' lies within R of the camera origin (ods_cull_bounds),
// and a ray from origin' meets the root box (the sphere) only if the same ray from the origin meets the box grown by R on every axis (the
// sphere grown by R).  So the panorama test runs from the origin with the grown box and sphere, on the strip's eye row, with alpha widened
// by delta; the sphere's growth of line_misses_sphere is taken at distance L + R.
template <bool kRegion, bool kPano = false, bool kOds = false>
__device__ __forceinline__ void miss_cull_body(const FrameArgs& fa, uint8_t* __restrict__ mask, const RenderRegion* rg, const Projection* pj = nullptr,
                                               const OdsParams* od = nullptr)
{
    __shared__ double3 planes[kCullPlanes];
    __shared__ int n_planes;
    const vpt_camera& cam = fa.cam;
    const FrameGeom& g = fa.geom;
    const double3 o = make_double3(cam.origin.x, cam.origin.y, cam.origin.z);
    double pmin[3], pmax[3];
    bool ok;
    if constexpr (kPano || kOds) ok = cam.lens_radius == 0.0f;
    else ok = pinhole_camera(cam);
    for (int a = 0; a < 3; ++a) {
        pmin[a] = fa.scene->root_pmin[a]; pmax[a] = fa.scene->root_pmax[a];
        ok = ok && isfinite(pmin[a]) && isfinite(pmax[a]) && pmin[a] <= pmax[a];       // an empty or broken root box culls nothing
    }
    OdsCullBounds ob; ob.R = 0.0; ob.delta = 0.0;
    if constexpr (kOds) {
        ob = ods_cull_bounds(cam, *od);
        ok = ok && ob.R >= 0.0;
        for (int a = 0; a < 3; ++a) { pmin[a] -= ob.R; pmax[a] += ob.R; }
    }
    if (threadIdx.x == 0) n_planes = 0;
    __syncthreads();
    if (ok && threadIdx.x < kCullPlanes) {
        const int t = threadIdx.x;
        double3 n = make_double3(0.0, 0.0, 0.0);
        if (t < 6) {
            const double s = (t & 1) ? -1.0 : 1.0;
            if (t >> 1 == 0) n.x = s; else if (t >> 1 == 1) n.y = s; else n.z = s;
        } else {
            int i = 0, k = (t - 6) >> 1;                          // pair k of the 28 pairs i < j of box corners
            while (k >= 7 - i) { k -= 7 - i; ++i; }
            const double3 a = box_corner(pmin, pmax, i, o), b = box_corner(pmin, pmax, i + 1 + k, o);
            const double s = ((t - 6) & 1) ? -1.0 : 1.0;
            n = make_double3(s * (a.y * b.z - a.z * b.y), s * (a.z * b.x - a.x * b.z), s * (a.x * b.y - a.y * b.x));
        }
        const double ln = len_d(n);
        bool keep = ln > 0.0;
        if (keep) {
            n = make_double3(n.x / ln, n.y / ln, n.z / ln);
            for (int i = 0; i < 8; ++i) { const double3 c = box_corner(pmin, pmax, i, o); keep = keep && dot_d(n, c) >= -kCullPlaneTol * len_d(c); }
        }
        if (keep) planes[atomicAdd(&n_planes, 1)] = n;
    }
    __syncthreads();

    // one thread per strip of kCullStrip pixels of one row: x0 .. x1 - 1
    int lr, x0;
    if constexpr (kRegion) {
        const int sx0 = rg->x0 / kCullStrip, strips_x = (rg->x1 + kCullStrip - 1) / kCullStrip - sx0;
        const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
        if (t >= (uint32_t)((rg->lr1 - rg->lr0) * strips_x)) return;
        const int r = (int)(t / (uint32_t)strips_x);
        lr = rg->lr0 + r; x0 = (sx0 + (int)(t - (uint32_t)r * (uint32_t)strips_x)) * kCullStrip;
    } else {
        const int strips_x = (g.width + kCullStrip - 1) / kCullStrip;
        const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
        if (t >= (uint32_t)(g.local_rows * strips_x)) return;
        lr = (int)(t / (uint32_t)strips_x); x0 = (int)(t - (uint32_t)lr * (uint32_t)strips_x) * kCullStrip;
    }
    const int x1 = min(x0 + kCullStrip, g.width);
    const int y = global_row(g, lr);
    bool culled = false;
    const SphereRec sph = load_sphere(fa.sphere);
    const double3 sa = make_double3(sph.center.x - o.x, sph.center.y - o.y, sph.center.z - o.z);
    const double L2 = dot_d(sa, sa), r2 = kOds ? ods_grown_r2(sph.radius, L2, ob.R) : 1.02 * (double)sph.radius * (double)sph.radius + 2e-3 * L2 + 1e-6;
    if constexpr (kOds) {
        if (ok && y < g.height && L2 > r2) {
            // the strip's eye row, as ods_camera takes it (one strip lies in one row, so in one eye)
            vpt_u2 re = fa.kp.resolution;
            int ye = y;
            if (od->layout == kOdsOverUnder) { re.y = fa.kp.resolution.y >> 1; if (y >= (int)re.y) ye = y - (int)re.y; }
            Projection pe; pe.kind = kProjOds; pe.hfov = od->hfov; pe.vfov = od->vfov;
            culled = pano_strip_culled<true>(cam, pe, re, x0, x1, ye, planes, n_planes, sa, L2, r2, ob.delta);
        }
    } else
    if constexpr (kPano) {
        if (ok && y < g.height && L2 > r2) culled = pano_strip_culled(cam, *pj, fa.kp.resolution, x0, x1, y, planes, n_planes, sa, L2, r2);
    } else
    if (ok && y < g.height && L2 > r2) {                         // (the comparison is false for a NaN sphere)
        // (b): D from the corners of the strip's jitter range: x0 + 0 .. (x1 - 1) + 1 = x1 + 0 (both exact), y + 0 .. y + 1
        double lo[3], hi[3], big = 0.0;
        for (int k = 0; k < 4; ++k) {
            const float3 b = camera_b0(cam, fa.kp.resolution, (k & 1) ? x1 : x0, y, 0.0f, (k & 2) ? 1.0f : 0.0f);
            const double c[3] = {b.x, b.y, b.z};
            for (int a = 0; a < 3; ++a) {
                lo[a] = k ? fmin(lo[a], c[a]) : c[a]; hi[a] = k ? fmax(hi[a], c[a]) : c[a];
                big = fmax(big, fabs(c[a]));
            }
        }
        bool signs = true;
        for (int a = 0; a < 3; ++a) signs = signs && (lo[a] > kCullSignMargin * big || hi[a] < -kCullSignMargin * big);
        if (signs) {
            const double3 mid = make_double3((lo[0] + hi[0]) / 2, (lo[1] + hi[1]) / 2, (lo[2] + hi[2]) / 2);
            const double3 half = make_double3((hi[0] - lo[0]) / 2, (hi[1] - lo[1]) / 2, (hi[2] - lo[2]) / 2);
            // |d| and the angle to a fixed axis are convex / quasi-convex on D: their largest values are at its corners
            const double ml = len_d(mid);
            const double3 f = make_double3(mid.x / ml, mid.y / ml, mid.z / ml);
            double dmax = 0.0, cos_theta = 1.0;                  // theta: the half-angle of the cone around f that holds D
            for (int i = 0; i < 8; ++i) {
                const double3 d = make_double3((i & 1) ? hi[0] : lo[0], (i & 2) ? hi[1] : lo[1], (i & 4) ? hi[2] : lo[2]);
                const double dl = len_d(d);
                dmax = fmax(dmax, dl);
                cos_theta = fmin(cos_theta, dot_d(f, d) / dl);
            }
            // (c)
            bool box_miss = false;
            for (int k = 0; k < n_planes && !box_miss; ++k) {
                const double3 n = planes[k];
                box_miss = dot_d(mid, n) + half.x * fabs(n.x) + half.y * fabs(n.y) + half.z * fabs(n.z) + kCullSlack * dmax < 0.0;
            }
            // (d): the angle beta between f and the sphere's centre exceeds gamma = theta + alpha + kCullSlack (alpha: the grown sphere's
            // angular radius), compared through cosines -- gamma stays below pi (theta < pi / 2 for D inside one octant, alpha < pi / 2)
            // unless sin(gamma) comes out negative, and then nothing is culled
            if (box_miss) {
                const double st = sqrt(fmax(0.0, 1.0 - cos_theta * cos_theta));
                const double sa_ = sqrt(r2 / L2), ca = sqrt(1.0 - r2 / L2);
                const double c1 = cos_theta * ca - st * sa_, s1 = st * ca + cos_theta * sa_;
                const double cs = 0.9999995000000417, ss = 9.999998333333417e-4;      // cos, sin of kCullSlack
                const double cg = c1 * cs - s1 * ss, sg = s1 * cs + c1 * ss;
                culled = sg > 0.0 && dot_d(f, sa) / sqrt(L2) < cg;
            }
        }
    }
    uint8_t* m = mask + (size_t)lr * g.width;
    for (int x = x0; x < x1; ++x) m[x] = culled ? 1 : 0;
}

__global__ void __launch_bounds__(256)
k_miss_cull(const FrameArgs fa, uint8_t* __restrict__ mask) { miss_cull_body<false>(fa, mask, nullptr); }

__global__ void __launch_bounds__(256)
k_miss_cull_region(const FrameArgs fa, uint8_t* __restrict__ mask, const RenderRegion rg) { miss_cull_body<true>(fa, mask, &rg); }

__global__ void __launch_bounds__(256)
k_miss_cull_equirect(const FrameArgs fa, uint8_t* __restrict__ mask, const Projection pj) { miss_cull_body<false, true>(fa, mask, nullptr, &pj); }

__global__ void __launch_bounds__(256)
k_miss_cull_region_equirect(const FrameArgs fa, uint8_t* __restrict__ mask, const RenderRegion rg, const Projection pj)
{
    miss_cull_body<true, true>(fa, mask, &rg, &pj);
}

__global__ void __launch_bounds__(256)
k_miss_cull_ods(const FrameArgs fa, uint8_t* __restrict__ mask, const OdsParams od) { miss_cull_body<false, false, true>(fa, mask, nullptr, nullptr, &od); }

__global__ void __launch_bounds__(256)
k_miss_cull_region_ods(const FrameArgs fa, uint8_t* __restrict__ mask, const RenderRegion rg, const OdsParams od)
{
    miss_cull_body<true, false, true>(fa, mask, &rg, nullptr, &od);
}


// =====================================================================================================
// k_resolve
// =====================================================================================================
// kSky 1: direct integrator with environment_type == 0 (Bruneton sky lookup, `atmo` is the caller's AtmosphereParameters);
// kSky 2: volumetric path integrator, which always ends on the sky (:1752); kSky 0: HDRI environment -- that variant
// takes a 16-byte dummy so it keeps its small parameter block and register budget.
struct NoSky { int pad[4]; };
struct PeerFlagPtrs { unsigned long long* p[kMaxPeers]; };

template <int kSky> using SkyArg = typename std::conditional<kSky != 0, vpt_atmosphere, NoSky>::type;

// The deep slice of a sample of depth d: the k with z[k] <= d < z[k + 1] (or z[n] = +inf), -1 when d is not > 0 (a miss, NaN) or lies
// outside [z[0], z[n]).  Binary search over the bounds in the parameter block.
__device__ __forceinline__ int deep_slice(const DeepSlices& dp, const float d)
{
    if (!(d > 0.0f) || !(d >= dp.z[0])) return -1;
    int lo = 0, hi = dp.n + 1;                                  // z[lo] <= d < z[hi] (z[n + 1] standing for +inf)
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (dp.z[mid] <= d) lo = mid; else hi = mid;
    }
    if (lo < dp.n) return lo;
    return isinf(dp.z[dp.n]) ? dp.n - 1 : -1;                   // d >= z[n]: only d = +inf under an open last slice
}
// One pass of a deep slice's running means {colour, coverage} with colour sample s and coverage sample c: accum's rule and arithmetic,
// written as the AOVs' (iteration 0 assigns, iteration < max_interactions updates x + (s - x) / (iteration + 1), later passes keep x)
__device__ __forceinline__ float4 deep_step(const float4 x, const float3 s, const float c, const uint32_t iteration, const uint32_t max_interactions)
{
    if (iteration == 0) return make_float4(s.x, s.y, s.z, c);
    if (iteration < max_interactions) {
        float3 v = f3(x.x, x.y, x.z);
        float w = x.w;
        v = v + (s - v) / (float)(iteration + 1);
        w = w + (c - w) / (float)(iteration + 1);
        return make_float4(v.x, v.y, v.z, w);
    }
    return x;
}

// The deep slices of one pixel during a chunk (resolve_pixel, kDeep).  K running means do not fit in registers, so each stays in its buffer
// and is updated lazily.  A pass that puts no sample in slice k updates it by x + (0 - x) / (iteration + 1), which needs nothing but x,
// so those updates wait until a sample lands in the slice (or the guard replaces a sample: then every slice takes a pass) and the end of
// the chunk, where every slice catches up.  done[k] = the passes of the chunk applied to slice k so far (a chunk that samples has at most
// 64 passes; one that samples nothing lands no sample, so done[] stays 0 there).
// The deep instantiations of resolve_pixel keep only the slices and store nothing else; launch_resolve runs the frame's own resolve kernel
// after them.  (Computing the slices inside that kernel moved accum and raw by an ulp in some frames: nvcc contracts the unpinned sky and
// tonemap arithmetic differently once the slice code is in the kernel, inlined or behind a call.)
struct DeepPixel { uint32_t lp, n_local, it0, max_interactions; };

// The instance mattes (section 8l) are the same running means with another bin: the instantiations whose pack ends with a Mattes run these
// functions on it (`Bins` = DeepSlices or Mattes; both have out and n).
// the bin of pass p's sample of depth d: its deep slice, or the matte its id maps to (the id plane is read only where d > 0, where the trace
// kernel wrote it); -1: none
__device__ __forceinline__ int sample_bin(const DeepSlices& dp, const float d, const DeepPixel&, const int) { return deep_slice(dp, d); }
__device__ __forceinline__ int sample_bin(const Mattes& mt, const float d, const DeepPixel& px, const int p)
{
    if (!(d > 0.0f)) return -1;
    const uint32_t id = mt.id[(size_t)p * px.n_local + px.lp];
    if (id == kMatteSphereId) return mt.sphere;
    return id < mt.n_ids ? (int)mt.map[id] : -1;
}

// slice k's means after the chunk's passes before `upto`, none of which since done[k] put a sample in it (at iteration 0 the zero sample
// is assigned, so the buffer is not read)
template <class Bins>
__device__ __forceinline__ float4 deep_catch_up(const Bins& dp, const uint8_t* done, const DeepPixel& px, const int k, const int upto)
{
    int q = done[k];
    float4 x;
    if (q < upto && px.it0 + (uint32_t)q == 0) { x = make_float4(0.f, 0.f, 0.f, 0.f); ++q; }
    else x = dp.out[(size_t)k * px.n_local + px.lp];
    for (; q < upto && px.it0 + (uint32_t)q < px.max_interactions; ++q) x = deep_step(x, f3(0.f), 0.0f, px.it0 + (uint32_t)q, px.max_interactions);
    return x;
}

// pass p of the chunk with the sample `value` (as it entered accum) of depth `depth`: its slice takes (value, 1) as the volume AOV takes
// it; a sample the guard replaced gives every slice its own mean as colour (at iteration 0: the buffer's previous content) and its slice
// the coverage 1 (coverage is not guarded)
template <class Bins>
__device__ __forceinline__ void deep_pass(const Bins& dp, uint8_t* done, const DeepPixel px, const int p, const float3 value, const float depth,
                                          const bool guarded)
{
    const uint32_t iteration = px.it0 + (uint32_t)p;
    const int b = sample_bin(dp, depth, px, p);
    if (guarded) {
        for (int k = 0; k < dp.n; ++k) {
            const float4 x = deep_catch_up(dp, done, px, k, p);
            dp.out[(size_t)k * px.n_local + px.lp] = deep_step(x, f3(x.x, x.y, x.z), k == b ? 1.0f : 0.0f, iteration, px.max_interactions);
            done[k] = (uint8_t)(p + 1);
        }
    } else if (b >= 0) {
        dp.out[(size_t)b * px.n_local + px.lp] = deep_step(deep_catch_up(dp, done, px, b, p), value, 1.0f, iteration, px.max_interactions);
        done[b] = (uint8_t)(p + 1);
    }
}

// the end of a chunk of n_passes passes: every slice catches up
template <class Bins>
__device__ __forceinline__ void deep_end(const Bins& dp, const uint8_t* done, const DeepPixel px, const int n_passes)
{
    for (int k = 0; k < dp.n; ++k)
        if (done[k] < n_passes) dp.out[(size_t)k * px.n_local + px.lp] = deep_catch_up(dp, done, px, k, n_passes);
}

// The adaptive rule's arithmetic (DESIGN.md section 8a), one code site for every k_resolve_adaptive instantiation and
// k_debug_adapt_pass.  Written in the round-to-nearest intrinsics of vpt_math.cuh in a fixed order, so that --use_fast_math neither
// contracts it differently per instantiation nor turns the divisions and the root into approximations; they compile to .rn.ftz.
// Welford step with the sample v as it entered the running mean:  Y = fma(0.0722, b, fma(0.2126, r, 0.7152 g));  n += 1;
// d = Y - mean;  mean += d / n;  M2 += d (Y - mean)  (a product and a sum, not an fma).
__device__ __forceinline__ void adapt_welford(float& wn, float& wmean, float& wm2, const float3 v)
{
    const float lum = pfma(0.0722f, v.z, pfma(0.2126f, v.x, pmul(0.7152f, v.y)));
    wn = padd(wn, 1.0f);
    const float d = psub(lum, wmean);
    wmean = padd(wmean, __fdiv_rn(d, wn));
    wm2 = padd(wm2, pmul(d, psub(lum, wmean)));
}
// err = sqrt(M2 / (n (n-1))) / max(mean, 1e-3), +Inf while n < 2 (a NaN mean takes the floor: fmaxf returns the other operand)
__device__ __forceinline__ float adapt_err(const float wn, const float wmean, const float wm2)
{
    if (!(wn >= 2.0f)) return INFINITY;
    return __fdiv_rn(__fsqrt_rn(__fdiv_rn(wm2, pmul(wn, psub(wn, 1.0f)))), fmaxf(wmean, kAdaptMeanFloor));
}

// One pixel of k_resolve (local pixel lp, local row lr, global row y).  kAdaptive (k_resolve_adaptive): the same running mean, plus the
// pixel's Welford state of the sample luminance and its pass count / relative error; no peer exchange.  kAov: also the running means of
// the compositing AOVs in `aov` (DESIGN.md section 8c).  kGroups: also the running means of the light groups in `lg` (section 8d).
// kPano (k_resolve_equirect, ...; HDRI frames): a culled pixel's miss samples are the equirectangular rays of the projection `pj`.
// kDeep: the deep slices in `dp` (section 8h), updated lazily in their buffer, and no other store (see deep_pass); with Bins = Mattes the
// instance mattes (section 8l) in their place.
template <int kSky, bool kAdaptive, bool kAov, bool kGroups = false, bool kPano = false, bool kDeep = false, bool kOds = false,
          class Bins = DeepSlices>
__device__ __forceinline__ void resolve_pixel(const FrameArgs& fa, const SkyArg<kSky>& atmo, const int n_passes, const int sampled,
                                              const int write_display, const PeerFrames& peers, const uint32_t lp, const int lr, const int y,
                                              const AdaptArgs* ad, const AovBuffers* aov, const LightGroups* lg = nullptr,
                                              const Projection* pj = nullptr, const Bins* dp = nullptr, const OdsParams* od = nullptr)
{
    const FrameGeom& g = fa.geom;
    const vpt_kernel_params& kp = fa.kp;
    const vpt_camera& cam = fa.cam;

    float3* accum_buf = reinterpret_cast<float3*>(kp.accum_buffer);
    float3* cost_buf = reinterpret_cast<float3*>(kp.cost_buffer);
    float*  depth_buf = reinterpret_cast<float*>(kp.depth_buffer);
    // output buffers are indexed by local pixel (== global pixel index for a single rank)
    float3 accum = f3(0.f), costv = f3(0.f); float depthv = 0.f;
    const bool have_prev = kp.iteration > 0;
    if (have_prev || !sampled) { accum = accum_buf[lp]; costv = cost_buf[lp]; depthv = depth_buf[lp]; }
    float tr = .0f;

    // adaptive: Welford state {n, mean, M2} of the luminance of every sample of this pixel
    float wn = 0.f, wmean = 0.f, wm2 = 0.f;
    if constexpr (kAdaptive) { if (have_prev) { const float4 st = ad->stat[lp]; wn = st.x; wmean = st.y; wm2 = st.z; } }
    // AOVs: alpha = mean of [depth > 0], volume = mean of the sample where depth > 0 and +0 elsewhere; read exactly when accum is
    float alphav = 0.f; float3 volv = f3(0.f);
    if constexpr (kAov) {
        if (have_prev || !sampled) { if (aov->alpha) alphav = aov->alpha[lp]; if (aov->volume) volv = aov->volume[lp]; }
    }
    // light groups: the running mean of each class, read exactly when accum is (a null output is kept at 0 and never stored)
    float3 gm[kLightGroups];
    if constexpr (kGroups) {
        #pragma unroll
        for (int k = 0; k < kLightGroups; ++k) gm[k] = ((have_prev || !sampled) && lg->out[k]) ? lg->out[k][lp] : f3(0.f);
    }
    // deep slices: the passes of the chunk applied to each slice so far (deep_pass)
    uint8_t done[kDeep ? kDeepMaxSlices : 1] = {};
    const DeepPixel dpx{lp, (uint32_t)g.n_local, kp.iteration, kp.max_interactions};
    // compact records (HDRI frames traced by a lean kernel, planeB null): one float4 per sample
    const bool compact = kSky == 0 && !fa.planeB;
    // a pixel culled by k_miss_cull has no records: every sample is the pinhole miss k_generate would have stored, direction rebuilt from
    // the chunk's jitter table, origin = the camera's
    const int px = (int)(lp - (uint32_t)lr * (uint32_t)g.width);
    // (HDRI frames only: the host hands the sky variants no mask -- their sky model is not written in pinned arithmetic, and with a second
    // source of env_pos in this function nvcc compiled it otherwise in some instantiations, which moved bits between them)
    const bool culled = kSky == 0 && sampled && fa.miss_mask && fa.miss_mask[lp];
    // one pass of the running mean; A (and B, C for a hit sample) are the pass's plane records, loaded by the caller.  Compact records:
    // B.x carries tr of a hit sample of the chunk's last pass when the display / raw words are written, C is unused.
    auto one_pass = [&](const int p, const float4 A, const float4 B, const float4 C) {
        const uint32_t iteration = kp.iteration + (uint32_t)p;
        float3 value = f3(1.0f);                                // WHITE when nothing is sampled (:2248)
        float depth = .0f;
        tr = .0f;
        // light-group samples; a pass that samples nothing gives its WHITE to the environment
        float3 gs[kLightGroups];
        if constexpr (kGroups) { gs[LG_SUN] = gs[LG_POINT] = gs[LG_EMISSION] = f3(0.f); gs[LG_ENVIRONMENT] = f3(1.0f); }
        if (sampled) {
            const size_t s = (size_t)p * g.n_local + lp;
            const float3 ray_dir = f3(A.x, A.y, A.z);
            float3 beta = f3(1.0f), L = f3(0.0f);
            const bool hit = __float_as_uint(A.w) != kMissSentinel;
            if (compact) {
                // the trace kernel finished a hit sample; a miss sees the environment along its direction
                if (hit) { L = f3(A.x, A.y, A.z); depth = A.w; tr = B.x; }
                else L = hdri_radiance((cudaTextureObject_t)kp.env_tex, ld3(kp.sky_color), ray_dir, L, beta);
            } else if (hit) {                                    // hit sample: the trace kernel wrote planes A, B, C (and D)
                beta = f3(C.x, C.y, C.z); L = f3(B.x, B.y, B.z);
                depth = B.w; tr = A.w;
            }
            if constexpr (kGroups) {
                // (records are wide: the host never hands these instantiations compact ones).  A hit sample's in-path sums: the generic
                // kernels' group planes, or for a lean kernel its L, which only the sun fed.  A miss is all environment.
                gs[LG_ENVIRONMENT] = f3(0.f);
                if (hit) {
                    if (lg->planes) {
                        const float* q = lg->planes + s;
                        const size_t n = lg->stride;
                        #pragma unroll
                        for (int k = 0; k < (kSky == 2 ? 4 : 3); ++k) gs[k] = f3(q[(3 * k) * n], q[(3 * k + 1) * n], q[(3 * k + 2) * n]);
                    } else gs[LG_SUN] = L;
                }
            }
            if constexpr (kSky == 0) {
                if constexpr (kGroups) {                        // hdri_radiance with L and with 0, from one look-up
                    const float3 t = hdri_product((cudaTextureObject_t)kp.env_tex, ld3(kp.sky_color), ray_dir, beta);
                    L = hdri_finish(t, L);
                    gs[LG_ENVIRONMENT] = hdri_finish(t, f3(0.f));
                } else
                if (!compact) L = hdri_radiance((cudaTextureObject_t)kp.env_tex, ld3(kp.sky_color), ray_dir, L, beta);
            } else if constexpr (kSky == 1) {
                // precomputed sky seen from env_pos along the final direction (:1838-1841)
                const float4 D = fa.planeD[s];
                if constexpr (kGroups) {
                    // the same fma as the instantiation without groups, once with L and once with 0 (pinned: the product has two uses)
                    const float3 P = sample_atmosphere(atmo, kp.azimuth, kp.elevation, f3(D.x, D.y, D.z), ray_dir) * beta * kp.sky_mult;
                    L = pfma3(P, ld3(kp.sky_color), L);
                    gs[LG_ENVIRONMENT] = pfma3(P, ld3(kp.sky_color), f3(0.f));
                } else
                L += sample_atmosphere(atmo, kp.azimuth, kp.elevation, f3(D.x, D.y, D.z), ray_dir) * beta * kp.sky_mult * ld3(kp.sky_color);
            } else if constexpr (kSky == 2) {
                const float4 D = fa.planeD[s];                       // env_pos or the last path position (:1750-1752)
                if constexpr (kGroups) {
                    // the in-path sky sum first, then the end-of-path sky, in the beauty's order
                    const float3 sa = sample_atmosphere(atmo, kp.azimuth, kp.elevation, f3(D.x, D.y, D.z), ray_dir);
                    L = pfma3(beta, sa, L);
                    gs[LG_ENVIRONMENT] = pfma3(beta, sa, gs[LG_ENVIRONMENT]);
                } else
                L += beta * sample_atmosphere(atmo, kp.azimuth, kp.elevation, f3(D.x, D.y, D.z), ray_dir);
            }
            tr = fminf(tr, 1.0f);
            value = L;
        }
        // NaN / Inf guard (:2263-2264): the sample becomes accum_buffer[idx].  At iteration 0 (the call's first pass) that is the buffer's
        // previous content, which was not loaded; the AOVs and groups take their own buffers' previous content likewise.
        bool guarded = false;                                   // AOVs / groups only, apart from the guard: the other instantiations keep their code
        if constexpr (kAov || kGroups || kDeep) guarded = any_nan(value) || any_inf(value);
        if (any_nan(value) || any_inf(value)) {
            if (iteration == 0) {
                accum = accum_buf[lp];
                if constexpr (kAov) { if (aov->volume) volv = aov->volume[lp]; }
                if constexpr (kGroups) {
                    #pragma unroll
                    for (int k = 0; k < kLightGroups; ++k) if (lg->out[k]) gm[k] = lg->out[k][lp];
                }
            }
            value = accum;
        }
        if (isnan(tr) || isinf(tr)) tr = 1.0f;

        float aof = 1 / cam.lens_radius;
        aof = clampf(aof, .0f, 3.402823466e+38F);
        if (cam.viz_dof) {
            if (depth > (cam.focus_dist + aof)) value = lerp3(value, f3(1.f, 0.f, 0.f), 0.5f);
            if (depth < (cam.focus_dist - aof)) value = lerp3(value, f3(0.f, 0.f, 1.f), 0.5f);
            if (depth > (cam.focus_dist - aof) && depth < (cam.focus_dist + aof)) value = lerp3(value, f3(0.f, 1.f, 0.f), 0.5f);
        }

        if (iteration == 0) { accum = value; costv = f3(0.f); depthv = depth; }
        else if (iteration < kp.max_interactions) {
            accum = accum + (value - accum) / (float)(iteration + 1);
            costv = costv + (f3(0.f) - costv) / (float)(iteration + 1);
            depthv = depthv + (depth - depthv) / (float)(iteration + 1);
        }
        if constexpr (kAov) {
            // the reference's collision decision of the camera ray (a NaN depth counts as none); selects, so a miss adds an exact +0.
            // A sample the guard replaced leaves the volume mean where it is, as the guard leaves accum.
            const bool c = depth > 0.0f;
            const float as = c ? 1.0f : 0.0f;
            const float3 vs = guarded ? volv : (c ? value : f3(0.f));
            if (iteration == 0) { alphav = as; volv = vs; }
            else if (iteration < kp.max_interactions) {
                alphav = alphav + (as - alphav) / (float)(iteration + 1);
                volv = volv + (vs - volv) / (float)(iteration + 1);
            }
        }
        if constexpr (kGroups) {
            // taken before the viz_dof tint; a sample the guard replaced leaves every group at its own mean
            #pragma unroll
            for (int k = 0; k < kLightGroups; ++k) {
                const float3 gv = guarded ? gm[k] : gs[k];
                if (iteration == 0) gm[k] = gv;
                else if (iteration < kp.max_interactions) gm[k] = gm[k] + (gv - gm[k]) / (float)(iteration + 1);
            }
        }
        if constexpr (kDeep) deep_pass(*dp, done, dpx, p, value, depth, guarded);
        if constexpr (kAdaptive) adapt_welford(wn, wmean, wm2, value);   // the sample as it entered the mean (after the NaN guard and the tint)
    };
    const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (culled) {
        // two loops, so the one over the records keeps the code (and register budget) it had without the cull
        for (int p = 0; p < n_passes; ++p) {
            const float2 j = __ldg(fa.bn_table + (size_t)p * 65536 + (y % 256) * 256 + px % 256);
            float3 d;
            if constexpr (kOds) d = normalize(camera_b0(ods_camera(cam, *od, kp.resolution, px, y, j.x, j.y).cam, kp.resolution, px, y, j.x, j.y));
            else if constexpr (kPano) d = normalize(pano_b0(cam, *pj, kp.resolution, px, y, j.x, j.y));
            else d = pinhole_dir(cam, kp.resolution, px, y, j.x, j.y);
            one_pass(p, make_float4(d.x, d.y, d.z, __uint_as_float(kMissSentinel)), zero4, zero4);
        }
    } else {
        for (int p = 0; p < n_passes; ++p) {
            float4 A = zero4, B = zero4, C = zero4;
            if (sampled) {
                const size_t s = (size_t)p * g.n_local + lp;
                A = fa.planeA[s];
                if (__float_as_uint(A.w) != kMissSentinel) {
                    if (compact) { if (write_display && p == n_passes - 1) B.x = fa.plane_tr[lp]; }
                    else { B = fa.planeB[s]; C = fa.planeC[s]; }
                }
            }
            one_pass(p, A, B, C);
        }
    }
    // the deep instantiations keep the slices and store nothing else: the frame's own resolve kernel runs after them (launch_resolve)
    if constexpr (kDeep) { deep_end(*dp, done, dpx, n_passes); return; }
    accum_buf[lp] = accum; cost_buf[lp] = costv; depth_buf[lp] = depthv;
    if constexpr (kAov) { if (aov->alpha) aov->alpha[lp] = alphav; if (aov->volume) aov->volume[lp] = volv; }
    if constexpr (kGroups) {
        #pragma unroll
        for (int k = 0; k < kLightGroups; ++k) if (lg->out[k]) lg->out[k][lp] = gm[k];
    }
    if constexpr (kAdaptive) {
        const float err = adapt_err(wn, wmean, wm2);
        ad->stat[lp] = make_float4(wn, wmean, wm2, err);
        ad->pass_count[lp] = kp.iteration + (uint32_t)n_passes;
        if (ad->rel_error) ad->rel_error[lp] = err;
    }

    if (write_display) {
        const Tonemapped tm = tonemap_display(accum, kp.exposure_scale);
        const unsigned int word = tm.word;
        reinterpret_cast<unsigned int*>(kp.display_buffer)[lp] = word;
        reinterpret_cast<float4*>(kp.raw_buffer)[lp] = make_float4(tm.val.x, tm.val.y, tm.val.z, tr);
        if (peers.n > 0 && peers.display[0]) {
            const size_t gp = (size_t)y * g.width + (lp - (uint32_t)lr * (uint32_t)g.width);
            #pragma unroll
            for (int p = 0; p < kMaxPeers; ++p) if (p < peers.n) peers.display[p][gp] = word;
        }
    }
    // multi-GPU exchange fused into the producer: this pixel's running mean goes to its global position in every rank's full frame
    if (peers.n > 0 && peers.accum[0]) {
        const size_t gp = (size_t)y * g.width + (lp - (uint32_t)lr * (uint32_t)g.width);
        #pragma unroll
        for (int p = 0; p < kMaxPeers; ++p) if (p < peers.n) { float* a = peers.accum[p] + 3 * gp; a[0] = accum.x; a[1] = accum.y; a[2] = accum.z; }
    }
}

// kAov / kGroups: the instantiations that also keep the compositing AOVs / the light groups take the AovBuffers / the LightGroups as
// more arguments (the pack `ext`, in that order, empty otherwise), so the kernels without them keep their parameter block.  The deep
// instantiations end the pack with a DeepSlices; it is the pack, not a template flag, that selects them, so every kernel without deep
// slices keeps its name as well.
__device__ __forceinline__ const AovBuffers* aov_of(const AovBuffers& a) { return &a; }
__device__ __forceinline__ const AovBuffers* aov_of(const AovBuffers& a, const LightGroups&) { return &a; }
__device__ __forceinline__ const LightGroups* lg_of(const AovBuffers&, const LightGroups& l) { return &l; }
__device__ __forceinline__ const AovBuffers* aov_of(const AovBuffers& a, const DeepSlices&) { return &a; }
__device__ __forceinline__ const AovBuffers* aov_of(const AovBuffers& a, const LightGroups&, const DeepSlices&) { return &a; }
__device__ __forceinline__ const LightGroups* lg_of(const LightGroups& l, const DeepSlices&) { return &l; }
__device__ __forceinline__ const LightGroups* lg_of(const AovBuffers&, const LightGroups& l, const DeepSlices&) { return &l; }
__device__ __forceinline__ const AovBuffers* aov_of(const AovBuffers& a, const Mattes&) { return &a; }
__device__ __forceinline__ const AovBuffers* aov_of(const AovBuffers& a, const LightGroups&, const Mattes&) { return &a; }
__device__ __forceinline__ const LightGroups* lg_of(const LightGroups& l, const Mattes&) { return &l; }
__device__ __forceinline__ const LightGroups* lg_of(const AovBuffers&, const LightGroups& l, const Mattes&) { return &l; }
// The matte instantiations end the pack with a Mattes instead: the deep code runs on it (bins_of), binned by id.
template <class... Ext> constexpr bool has_mattes = (std::is_same<Ext, Mattes>::value || ... || false);
template <class... Ext> constexpr bool has_deep = (std::is_same<Ext, DeepSlices>::value || ... || false) || has_mattes<Ext...>;
template <class... Ext> using bins_of = typename std::conditional<has_mattes<Ext...>, Mattes, DeepSlices>::type;
template <class B> __device__ __forceinline__ const B* deep_of(const B& d) { return &d; }
template <class B> __device__ __forceinline__ const B* deep_of(const AovBuffers&, const B& d) { return &d; }
template <class B> __device__ __forceinline__ const B* deep_of(const LightGroups&, const B& d) { return &d; }
template <class B> __device__ __forceinline__ const B* deep_of(const AovBuffers&, const LightGroups&, const B& d) { return &d; }

// The thread's pixel and its resolve_pixel, shared by k_resolve, k_resolve_equirect and k_resolve_ods (kProj: 0 the perspective camera,
// 1 the equirectangular projection `pj`, 2 the ODS projection `od`)
template <int kSky, bool kAov, bool kGroups, int kProj, class... Ext>
__device__ __forceinline__ void resolve_body(const FrameArgs& fa, const SkyArg<kSky>& atmo, const int n_passes, const int sampled,
                                             const int write_display, const PeerFrames& peers, const Projection* pj, const OdsParams* od,
                                             const Ext&... ext)
{
    const FrameGeom& g = fa.geom;
    const uint32_t lp = blockIdx.x * blockDim.x + threadIdx.x;
    if (lp >= (uint32_t)g.n_local) return;
    const int lr = lp / g.width;
    const int y = global_row(g, lr);
    if (y >= g.height) return;
    const AovBuffers* ap = nullptr;
    const LightGroups* gp = nullptr;
    const bins_of<Ext...>* dq = nullptr;
    if constexpr (kAov) ap = aov_of(ext...);
    if constexpr (kGroups) gp = lg_of(ext...);
    if constexpr (has_deep<Ext...>) dq = deep_of(ext...);
    resolve_pixel<kSky, false, kAov, kGroups, kProj == 1, has_deep<Ext...>, kProj == 2, bins_of<Ext...>>(fa, atmo, n_passes, sampled, write_display, peers, lp, lr, y,
                                                                                         nullptr, ap, gp, pj, dq, od);
}

template <int kSky, bool kAov = false, bool kGroups = false, class... Ext>
__global__ void __launch_bounds__(256)
k_resolve(const FrameArgs fa, const SkyArg<kSky> atmo, const int n_passes, const int sampled, const int write_display, const PeerFrames peers,
          const Ext... ext)
{
    static_assert(sizeof...(Ext) == (kAov ? 1 : 0) + (kGroups ? 1 : 0) + (has_deep<Ext...> ? 1 : 0),"k_resolve<kSky, kAov, kGroups> takes an AovBuffers if kAov, then a LightGroups if kGroups, then a DeepSlices for the deep slices");
    resolve_body<kSky, kAov, kGroups, 0>(fa, atmo, n_passes, sampled, write_display, peers, nullptr, nullptr, ext...);
}

// k_resolve over R only: one thread per pixel of R on this rank, region row by region row (rg.lr0 .. rg.lr1 - 1, columns rg.x0 .. rg.x1 - 1),
// so a warp reads and writes consecutive pixels of one row as k_resolve does.  Every pixel it visits is a pixel of R.  Shared by
// k_resolve_region and k_resolve_region_equirect.
template <int kSky, bool kAov, bool kGroups, int kProj, class... Ext>
__device__ __forceinline__ void resolve_region_body(const FrameArgs& fa, const SkyArg<kSky>& atmo, const int n_passes, const int sampled,
                                                    const int write_display, const PeerFrames& peers, const RenderRegion& rg, const Projection* pj,
                                                    const OdsParams* od, const Ext&... ext)
{
    const FrameGeom& g = fa.geom;
    const uint32_t w = (uint32_t)(rg.x1 - rg.x0);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= w * (uint32_t)(rg.lr1 - rg.lr0)) return;
    const uint32_t r = i / w;
    const int lr = rg.lr0 + (int)r;
    const uint32_t lp = (uint32_t)lr * (uint32_t)g.width + (uint32_t)rg.x0 + (i - r * w);
    const AovBuffers* ap = nullptr;
    const LightGroups* gp = nullptr;
    const bins_of<Ext...>* dq = nullptr;
    if constexpr (kAov) ap = aov_of(ext...);
    if constexpr (kGroups) gp = lg_of(ext...);
    if constexpr (has_deep<Ext...>) dq = deep_of(ext...);
    resolve_pixel<kSky, false, kAov, kGroups, kProj == 1, has_deep<Ext...>, kProj == 2, bins_of<Ext...>>(fa, atmo, n_passes, sampled, write_display, peers, lp, lr,
                                                                                         global_row(g, lr), nullptr, ap, gp, pj, dq, od);
}

template <int kSky, bool kAov = false, bool kGroups = false, class... Ext>
__global__ void __launch_bounds__(256)
k_resolve_region(const FrameArgs fa, const SkyArg<kSky> atmo, const int n_passes, const int sampled, const int write_display, const PeerFrames peers,
                 const RenderRegion rg, const Ext... ext)
{
    static_assert(sizeof...(Ext) == (kAov ? 1 : 0) + (kGroups ? 1 : 0) + (has_deep<Ext...> ? 1 : 0),"k_resolve_region<kSky, kAov, kGroups> takes an AovBuffers if kAov, then a LightGroups if kGroups, then a DeepSlices for the deep slices");
    resolve_region_body<kSky, kAov, kGroups, 0>(fa, atmo, n_passes, sampled, write_display, peers, rg, nullptr, nullptr, ext...);
}

// The equirectangular frames of the HDRI environment (sky 0): k_resolve, k_resolve_region and k_resolve_adaptive with the projection `pj` as
// one more argument, for the culled pixels' miss samples.  (Frames that end on the precomputed sky cull nothing and run k_resolve<1/2>.)
template <bool kAov = false, bool kGroups = false, class... Ext>
__global__ void __launch_bounds__(256)
k_resolve_equirect(const FrameArgs fa, const NoSky atmo, const int n_passes, const int sampled, const int write_display, const PeerFrames peers,
                   const Projection pj, const Ext... ext)
{
    static_assert(sizeof...(Ext) == (kAov ? 1 : 0) + (kGroups ? 1 : 0) + (has_deep<Ext...> ? 1 : 0),"k_resolve_equirect<kAov, kGroups> takes an AovBuffers if kAov, then a LightGroups if kGroups, then a DeepSlices for the deep slices");
    resolve_body<0, kAov, kGroups, 1>(fa, atmo, n_passes, sampled, write_display, peers, &pj, nullptr, ext...);
}

template <bool kAov = false, bool kGroups = false, class... Ext>
__global__ void __launch_bounds__(256)
k_resolve_region_equirect(const FrameArgs fa, const NoSky atmo, const int n_passes, const int sampled, const int write_display, const PeerFrames peers,
                          const RenderRegion rg, const Projection pj, const Ext... ext)
{
    static_assert(sizeof...(Ext) == (kAov ? 1 : 0) + (kGroups ? 1 : 0) + (has_deep<Ext...> ? 1 : 0),"k_resolve_region_equirect<kAov, kGroups> takes an AovBuffers if kAov, then a LightGroups if kGroups, then a DeepSlices for the deep slices");
    resolve_region_body<0, kAov, kGroups, 1>(fa, atmo, n_passes, sampled, write_display, peers, rg, &pj, nullptr, ext...);
}

// The ODS frames of the HDRI environment (sky 0): the same with the ODS projection `od`, whose culled pixels' miss samples are rebuilt from
// ods_camera (k_miss_cull_ods guarantees they took the pinhole order)
template <bool kAov = false, bool kGroups = false, class... Ext>
__global__ void __launch_bounds__(256)
k_resolve_ods(const FrameArgs fa, const NoSky atmo, const int n_passes, const int sampled, const int write_display, const PeerFrames peers,
              const OdsParams od, const Ext... ext)
{
    static_assert(sizeof...(Ext) == (kAov ? 1 : 0) + (kGroups ? 1 : 0) + (has_deep<Ext...> ? 1 : 0),"k_resolve_ods<kAov, kGroups> takes an AovBuffers if kAov, then a LightGroups if kGroups, then a DeepSlices for the deep slices");
    resolve_body<0, kAov, kGroups, 2>(fa, atmo, n_passes, sampled, write_display, peers, nullptr, &od, ext...);
}

template <bool kAov = false, bool kGroups = false, class... Ext>
__global__ void __launch_bounds__(256)
k_resolve_region_ods(const FrameArgs fa, const NoSky atmo, const int n_passes, const int sampled, const int write_display, const PeerFrames peers,
                     const RenderRegion rg, const OdsParams od, const Ext... ext)
{
    static_assert(sizeof...(Ext) == (kAov ? 1 : 0) + (kGroups ? 1 : 0) + (has_deep<Ext...> ? 1 : 0),"k_resolve_region_ods<kAov, kGroups> takes an AovBuffers if kAov, then a LightGroups if kGroups, then a DeepSlices for the deep slices");
    resolve_region_body<0, kAov, kGroups, 2>(fa, atmo, n_passes, sampled, write_display, peers, rg, nullptr, &od, ext...);
}

// 32x4 pixel tile and the lane's pixel in it, for the per-tile adaptive kernels (a warp covers one row of 32 pixels)
struct TilePixel { int x, lr; bool inside; };
__device__ __forceinline__ TilePixel tile_pixel(const FrameGeom& g, const int tile)
{
    const int tiles_x = (g.width + 31) / 32;
    const int ty = tile / tiles_x, tx = tile - ty * tiles_x;
    TilePixel t; t.x = tx * 32 + (int)(threadIdx.x & 31); t.lr = ty * 4 + (int)(threadIdx.x >> 5);
    t.inside = t.x < g.width && t.lr < g.local_rows && global_row(g, t.lr) < g.height;
    return t;
}

// One block of 128 per active tile: the running mean of the pixels that have not stopped, every pass of the chunk sampled; at the end of the
// chunk their display / raw words, pass count and relative error (so a pixel keeps those of the last pass it took).  kAov: as k_resolve.
template <int kSky, bool kAov, bool kGroups, int kProj, class... Ext>
__device__ __forceinline__ void resolve_adaptive_body(const FrameArgs& fa, const SkyArg<kSky>& atmo, const int n_passes, const AdaptArgs& ad,
                                                      const Projection* pj, const OdsParams* od, const Ext&... ext)
{
    const FrameGeom& g = fa.geom;
    const TilePixel t = tile_pixel(g, (int)__ldg(ad.tiles + blockIdx.x));
    if (!t.inside) return;
    const uint32_t lp = (uint32_t)t.lr * (uint32_t)g.width + (uint32_t)t.x;
    if (ad.stopped[lp]) return;
    const AovBuffers* ap = nullptr;
    const LightGroups* gp = nullptr;
    const bins_of<Ext...>* dq = nullptr;
    if constexpr (kAov) ap = aov_of(ext...);
    if constexpr (kGroups) gp = lg_of(ext...);
    if constexpr (has_deep<Ext...>) dq = deep_of(ext...);
    resolve_pixel<kSky, true, kAov, kGroups, kProj == 1, has_deep<Ext...>, kProj == 2, bins_of<Ext...>>(fa, atmo, n_passes, 1, 1, PeerFrames{}, lp, t.lr,
                                                                                        global_row(g, t.lr), &ad, ap, gp, pj, dq, od);
}

template <int kSky, bool kAov = false, bool kGroups = false, class... Ext>
__global__ void __launch_bounds__(128)
k_resolve_adaptive(const FrameArgs fa, const SkyArg<kSky> atmo, const int n_passes, const AdaptArgs ad, const Ext... ext)
{
    static_assert(sizeof...(Ext) == (kAov ? 1 : 0) + (kGroups ? 1 : 0) + (has_deep<Ext...> ? 1 : 0),"k_resolve_adaptive<kSky, kAov, kGroups> takes an AovBuffers if kAov, then a LightGroups if kGroups, then a DeepSlices for the deep slices");
    resolve_adaptive_body<kSky, kAov, kGroups, 0>(fa, atmo, n_passes, ad, nullptr, nullptr, ext...);
}

template <bool kAov = false, bool kGroups = false, class... Ext>
__global__ void __launch_bounds__(128)
k_resolve_adaptive_equirect(const FrameArgs fa, const NoSky atmo, const int n_passes, const AdaptArgs ad, const Projection pj, const Ext... ext)
{
    static_assert(sizeof...(Ext) == (kAov ? 1 : 0) + (kGroups ? 1 : 0) + (has_deep<Ext...> ? 1 : 0),"k_resolve_adaptive_equirect<kAov, kGroups> takes an AovBuffers if kAov, then a LightGroups if kGroups, then a DeepSlices for the deep slices");
    resolve_adaptive_body<0, kAov, kGroups, 1>(fa, atmo, n_passes, ad, &pj, nullptr, ext...);
}

template <bool kAov = false, bool kGroups = false, class... Ext>
__global__ void __launch_bounds__(128)
k_resolve_adaptive_ods(const FrameArgs fa, const NoSky atmo, const int n_passes, const AdaptArgs ad, const OdsParams od, const Ext... ext)
{
    static_assert(sizeof...(Ext) == (kAov ? 1 : 0) + (kGroups ? 1 : 0) + (has_deep<Ext...> ? 1 : 0),"k_resolve_adaptive_ods<kAov, kGroups> takes an AovBuffers if kAov, then a LightGroups if kGroups, then a DeepSlices for the deep slices");
    resolve_adaptive_body<0, kAov, kGroups, 2>(fa, atmo, n_passes, ad, nullptr, &od, ext...);
}

// =====================================================================================================
// k_motion_vectors: screen-space motion of each sample's first collision towards a second camera pose (DESIGN.md section 8o)
// =====================================================================================================
// The film projection pi_K of camera K (FilmCam, film_cam, film_project): vpt_film.cuh

// The accepted lens point of the rejection loop k_generate runs on the pixel's stream (two draws per trial through vanDerCorput in bases 2
// and 3): the radical inverses k_generate tabulates, computed by the same operations
__device__ __forceinline__ float2 lens_disk_point(Rng& rng)
{
    float2 p;
    do {
        const float a = van_der_corput<2>(rng);
        const float b = van_der_corput<3>(rng);
        p = make_float2(pfma(a, 2.0f, -1.0f), pfma(b, 2.0f, -1.0f));
    } while (pfma(p.x, p.x, pmul(p.y, p.y)) >= 1.0f);
    return p;
}

// The camera ray of pixel (x, global row y)'s sample on the Philox stream of `iteration` (the sample offset included), jitter j, as k_generate (kMotion: k_generate_motion) built it: the
// pinhole order where k_generate takes it, else the thin-lens order with the loop's lens point (and, under motion, the camera of the shutter
// draw that follows the loop)
template <bool kMotion>
__device__ __forceinline__ void sample_camera_ray(const FrameArgs& fa, const CameraMotion* mo, const int x, const int y, const uint32_t iteration,
                                                  const float2 j, float3& org, float3& dir)
{
    const vpt_camera& cam = fa.cam;
    const vpt_u2 res = fa.kp.resolution;
    Rng rng; rng.init((uint32_t)y * (uint32_t)fa.geom.width + (uint32_t)x, iteration, 0u);
    if constexpr (!kMotion) {
        const float3 b0 = camera_b0(cam, res, x, y, j.x, j.y);
        if (pinhole_camera(cam) && b0.x != 0.0f && b0.y != 0.0f && b0.z != 0.0f) { org = ld3(cam.origin); dir = normalize(b0); return; }
    }
    const float2 p = lens_disk_point(rng);
    vpt_camera mc;
    if constexpr (kMotion) mc = motion_camera(cam, *mo, rng.next());
    const vpt_camera& pc = kMotion ? mc : cam;
    const float3 rd = f3(pmul(cam.lens_radius, p.x), pmul(cam.lens_radius, p.y), 0.0f);
    const float3 offset = f3(pfma(pc.u.x, rd.x, pmul(pc.v.x, rd.y)), pfma(pc.u.y, rd.x, pmul(pc.v.y, rd.y)), pfma(pc.u.z, rd.x, pmul(pc.v.z, rd.y)));
    const float3 b0 = camera_b0(pc, res, x, y, j.x, j.y);
    org = f3(padd(pc.origin.x, offset.x), padd(pc.origin.y, offset.y), padd(pc.origin.z, offset.z));
    dir = normalize(f3(psub(b0.x, offset.x), psub(b0.y, offset.y), psub(b0.z, offset.z)));
}

// The depth word of pass p's record of local pixel lp (A.w of a compact record, B.w of a wide one); 0 for a miss and where `records` is false
// (a pixel k_miss_cull removed, or a pass that samples nothing: no record)
__device__ __forceinline__ float record_depth(const FrameArgs& fa, const int p, const uint32_t lp, const bool records, const bool compact)
{
    float depth = 0.0f;
    if (records) {
        const size_t s = (size_t)p * fa.geom.n_local + lp;
        const float4 a = fa.planeA[s];
        if (__float_as_uint(a.w) != kMissSentinel) depth = compact ? a.w : fa.planeB[s].w;
    }
    return depth;
}

// the camera ray of pixel (x, global row y)'s sample in pass p of the chunk (iteration = kp.iteration + p): the pass's jitter, the Philox
// stream of the sample offset + iteration
template <bool kMotion>
__device__ __forceinline__ void pass_camera_ray(const FrameArgs& fa, const CameraMotion* mo, const int x, const int y, const int p,
                                                const uint32_t iteration, float3& org, float3& dir)
{
    const float2 j = __ldg(fa.bn_table + (size_t)p * 65536 + (y % 256) * 256 + x % 256);
    sample_camera_ray<kMotion>(fa, mo, x, y, fa.sample_offset + iteration, j, org, dir);
}

// One pixel (local pixel lp, local row lr, global row y) over the chunk's passes.  Reads only each record's depth word (a miss, or a pixel
// k_miss_cull removed, has none: c = 0), rebuilds the camera ray of the samples with c and keeps the running means in accum's rule and
// arithmetic, written as the alpha AOV's, so z is alpha bit for bit.
template <bool kMotion>
__device__ __forceinline__ void motion_vectors_pixel(const FrameArgs& fa, const MotionVectors& mv, const CameraMotion* mo, const int n_passes,
                                                     const int sampled, const uint32_t lp, const int lr, const int y)
{
    const FrameGeom& g = fa.geom;
    const vpt_kernel_params& kp = fa.kp;
    const int x = (int)(lp - (uint32_t)lr * (uint32_t)g.width);
    const FilmCam A = film_cam(fa.cam.origin, fa.cam.lower_left_corner, fa.cam.horizontal, fa.cam.vertical);
    const FilmCam B = film_cam(mv.origin, mv.lower_left_corner, mv.horizontal, mv.vertical);
    float3 m = kp.iteration > 0 ? mv.out[lp] : f3(0.f);
    const bool records = sampled && !(fa.miss_mask && fa.miss_mask[lp]);
    const bool compact = !fa.planeB;
    for (int p = 0; p < n_passes; ++p) {
        const uint32_t iteration = kp.iteration + (uint32_t)p;
        const float depth = record_depth(fa, p, lp, records, compact);
        const bool c = depth > 0.0f;
        float vx = 0.0f, vy = 0.0f;
        if (c) {
            float3 org, dir;
            const float2 j = __ldg(fa.bn_table + (size_t)p * 65536 + (y % 256) * 256 + x % 256);
            sample_camera_ray<kMotion>(fa, mo, x, y, fa.sample_offset + iteration, j, org, dir);
            const float3 P = madd3(org, dir, depth);
            float2 pa, pb;
            if (film_project(A, P, kp.resolution, &pa) && film_project(B, P, kp.resolution, &pb)) { vx = psub(pb.x, pa.x); vy = psub(pb.y, pa.y); }
        }
        const float as = c ? 1.0f : 0.0f;
        if (iteration == 0) m = f3(vx, vy, as);
        else if (iteration < kp.max_interactions) {
            m.x = m.x + (vx - m.x) / (float)(iteration + 1);
            m.y = m.y + (vy - m.y) / (float)(iteration + 1);
            m.z = m.z + (as - m.z) / (float)(iteration + 1);
        }
    }
    mv.out[lp] = m;
}

// The pixel walkers of the per-pixel layer kernels (k_motion_vectors*, k_collision_aovs*): each calls f(lp, lr, y) for one pixel of the
// thread.  frame: every local pixel (padding rows are skipped); region: R's pixels on this rank, row by row as k_resolve_region walks them;
// adaptive: the pixels of the active tiles that have not stopped, as k_resolve_adaptive visits them.
template <class F>
__device__ __forceinline__ void frame_pixel(const FrameGeom& g, F&& f)
{
    const uint32_t lp = blockIdx.x * blockDim.x + threadIdx.x;
    if (lp >= (uint32_t)g.n_local) return;
    const int lr = lp / g.width;
    const int y = global_row(g, lr);
    if (y >= g.height) return;
    f(lp, lr, y);
}

template <class F>
__device__ __forceinline__ void region_pixel(const FrameGeom& g, const RenderRegion& rg, F&& f)
{
    const uint32_t w = (uint32_t)(rg.x1 - rg.x0);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= w * (uint32_t)(rg.lr1 - rg.lr0)) return;
    const uint32_t r = i / w;
    const int lr = rg.lr0 + (int)r;
    const uint32_t lp = (uint32_t)lr * (uint32_t)g.width + (uint32_t)rg.x0 + (i - r * w);
    f(lp, lr, global_row(g, lr));
}

template <class F>
__device__ __forceinline__ void adaptive_pixel(const FrameGeom& g, const AdaptArgs& ad, F&& f)
{
    const TilePixel t = tile_pixel(g, (int)__ldg(ad.tiles + blockIdx.x));
    if (!t.inside) return;
    const uint32_t lp = (uint32_t)t.lr * (uint32_t)g.width + (uint32_t)t.x;
    if (ad.stopped[lp]) return;
    f(lp, t.lr, global_row(g, t.lr));
}

__global__ void __launch_bounds__(256)
k_motion_vectors(const FrameArgs fa, const MotionVectors mv, const int n_passes, const int sampled)
{ frame_pixel(fa.geom, [&](uint32_t lp, int lr, int y) { motion_vectors_pixel<false>(fa, mv, nullptr, n_passes, sampled, lp, lr, y); }); }

__global__ void __launch_bounds__(256)
k_motion_vectors_region(const FrameArgs fa, const MotionVectors mv, const int n_passes, const int sampled, const RenderRegion rg)
{ region_pixel(fa.geom, rg, [&](uint32_t lp, int lr, int y) { motion_vectors_pixel<false>(fa, mv, nullptr, n_passes, sampled, lp, lr, y); }); }

__global__ void __launch_bounds__(128)
k_motion_vectors_adaptive(const FrameArgs fa, const MotionVectors mv, const int n_passes, const AdaptArgs ad)
{ adaptive_pixel(fa.geom, ad, [&](uint32_t lp, int lr, int y) { motion_vectors_pixel<false>(fa, mv, nullptr, n_passes, 1, lp, lr, y); }); }

__global__ void __launch_bounds__(256)
k_motion_vectors_motion(const FrameArgs fa, const MotionVectors mv, const int n_passes, const int sampled, const CameraMotion mo)
{ frame_pixel(fa.geom, [&](uint32_t lp, int lr, int y) { motion_vectors_pixel<true>(fa, mv, &mo, n_passes, sampled, lp, lr, y); }); }

__global__ void __launch_bounds__(256)
k_motion_vectors_region_motion(const FrameArgs fa, const MotionVectors mv, const int n_passes, const int sampled, const RenderRegion rg,
                               const CameraMotion mo)
{ region_pixel(fa.geom, rg, [&](uint32_t lp, int lr, int y) { motion_vectors_pixel<true>(fa, mv, &mo, n_passes, sampled, lp, lr, y); }); }

__global__ void __launch_bounds__(128)
k_motion_vectors_adaptive_motion(const FrameArgs fa, const MotionVectors mv, const int n_passes, const AdaptArgs ad, const CameraMotion mo)
{ adaptive_pixel(fa.geom, ad, [&](uint32_t lp, int lr, int y) { motion_vectors_pixel<true>(fa, mv, &mo, n_passes, 1, lp, lr, y); }); }

// =====================================================================================================
// k_collision_aovs: world position, density normal and albedo at each sample's first collision (DESIGN.md section 8q)
// =====================================================================================================
// The leaf of the octree that contains X (the descent oct_locate_or_skip takes, read from the flat tables), or -1 when X lies outside the
// root box or in an empty node
__device__ __forceinline__ int collision_leaf(const SceneTables& sc, const float3 X)
{
    if (!aabb_contains(sc.root_pmin, sc.root_pmax, X)) return -1;
    const OctInternal r = sc.internal[0];
    const int c1 = oct_child(r, X);
    if ((r.child_empty >> c1) & 1u) return -1;
    const OctInternal n1 = sc.internal[1 + c1];
    const int c2 = oct_child(n1, X);
    if ((n1.child_empty >> c2) & 1u) return -1;
    const OctInternal n2 = sc.internal[9 + c1 * 8 + c2];
    const int c3 = oct_child(n2, X);
    if ((n2.child_empty >> c3) & 1u) return -1;
    return c1 * 64 + c2 * 8 + c3;
}

// rho(X), the density the frame's tracker reads at X: volume 0 through the frame's sampler (brick pool, cell table or texture) in a
// single-volume scene, else the sum over the leaf list of the leaf that contains X (0 in no populated leaf)
__device__ __forceinline__ float collision_density(const FrameArgs& fa, const CollisionAovs& ca, const SceneTables& sc, const VolumeRec& vol0,
                                                   const float3 X)
{
    if (ca.brick_pool) {
        BrickArgs ba;
        ba.pool = ca.brick_pool; ba.dimx = ca.brick_dims[0]; ba.dimy = ca.brick_dims[1]; ba.dimz = ca.brick_dims[2];
        ba.nbx = (ba.dimx + 3) / 4; ba.nby = (ba.dimy + 3) / 4; ba.nbz = (ba.dimz + 3) / 4;
        float3 uvw;
        if (!volume_coord(vol0, X, uvw)) return 0.0f;
        return 0.0f + brick_sample_global<kBrickWeightMode>(uvw, ba);
    }
    if (fa.cell_table) return 0.0f + cell_density(fa, vol0, X);
    if (sc.single_volume) return 0.0f + volume_density(vol0, X);
    const int leaf = collision_leaf(sc, X);
    return leaf < 0 ? 0.0f : leaf_density(sc, vol0, leaf, X);
}

// The normal and albedo of a covered sample whose camera ray (org, dir) first collided at P.  The depth pass's own test on the ray tells the
// sphere from the volume: the sphere gives normalize(P - centre) and its colour (the reflectance the integrators' sphere branch multiplies
// the throughput by); the volume gives -grad rho / |grad rho| by central differences of step h (0 where |grad rho| is 0 or not finite) and
// the throughput factor scatter_event applies at an accepted collision at P.
__device__ __forceinline__ void collision_surface(const FrameArgs& fa, const CollisionAovs& ca, const float3 org, const float3 dir, const float3 P,
                                                  float3& n, float3& a)
{
    const vpt_kernel_params& kp = fa.kp;
    const SceneTables& sc = *fa.scene;
    const SphereRec sph = load_sphere(fa.sphere);
    float t_min;
    if (closest_object(sc, sph, org, dir, t_min) == 2) {
        n = normalize(P - sph.center);
        a = sph.color;
        return;
    }
    const VolumeRec& vol0 = sc.volumes[0];
    const float rho = collision_density(fa, ca, sc, vol0, P);
    if (ca.normal) {
        const float h = ca.step, inv2h = 1.0f / padd(h, h);
        const float gx = pmul(psub(collision_density(fa, ca, sc, vol0, f3(padd(P.x, h), P.y, P.z)),
                                   collision_density(fa, ca, sc, vol0, f3(psub(P.x, h), P.y, P.z))), inv2h);
        const float gy = pmul(psub(collision_density(fa, ca, sc, vol0, f3(P.x, padd(P.y, h), P.z)),
                                   collision_density(fa, ca, sc, vol0, f3(P.x, psub(P.y, h), P.z))), inv2h);
        const float gz = pmul(psub(collision_density(fa, ca, sc, vol0, f3(P.x, P.y, padd(P.z, h))),
                                   collision_density(fa, ca, sc, vol0, f3(P.x, P.y, psub(P.z, h)))), inv2h);
        const float g2 = pfma(gx, gx, pfma(gy, gy, pmul(gz, gz)));
        if (g2 > 0.0f && g2 <= VPT_M_INF) {                      // positive and finite
            const float r = -rsqrtf(g2);
            n = f3(pmul(gx, r), pmul(gy, r), pmul(gz, r));
        }
    }
    if (ca.albedo) {
        float3 Cd;
        if (sc.single_volume) Cd = fmax3(f3(0.0f), volume_color(vol0, P));
        else { const int leaf = collision_leaf(sc, P); Cd = leaf < 0 ? f3(0.0f) : leaf_color(sc, vol0, leaf, P); }
        const int index = int(floorf(fminf(fmaxf((rho * (1.0f / sc.max_extinction) * 255.0f / kp.emission_pivot), 0.0f), 255.0f)));
        const float3 density_color = reinterpret_cast<const float3*>(kp.density_color_texture)[index];
        a = (ld3(kp.albedo) * Cd * density_color / ld3(kp.extinction)) * float(kp.energy_inject);
    }
}

// One pixel over the chunk's passes, as motion_vectors_pixel: every record's depth word, the camera ray and the look-ups only for samples
// with c, the running means in accum's rule with the alpha AOV's expressions (so position.w is alpha bit for bit; a sample without c adds
// exact zeros)
template <bool kMotion>
__device__ __forceinline__ void collision_aovs_pixel(const FrameArgs& fa, const CollisionAovs& ca, const CameraMotion* mo, const int n_passes,
                                                     const int sampled, const uint32_t lp, const int lr, const int y)
{
    const FrameGeom& g = fa.geom;
    const vpt_kernel_params& kp = fa.kp;
    const int x = (int)(lp - (uint32_t)lr * (uint32_t)g.width);
    const bool prev = kp.iteration > 0;
    float4 mp = prev && ca.position ? ca.position[lp] : make_float4(0.f, 0.f, 0.f, 0.f);
    float3 mn = prev && ca.normal ? ca.normal[lp] : f3(0.f);
    float3 ma = prev && ca.albedo ? ca.albedo[lp] : f3(0.f);
    const bool records = sampled && !(fa.miss_mask && fa.miss_mask[lp]);
    const bool compact = !fa.planeB;
    for (int p = 0; p < n_passes; ++p) {
        const uint32_t iteration = kp.iteration + (uint32_t)p;
        const float depth = record_depth(fa, p, lp, records, compact);
        const bool c = depth > 0.0f;
        float3 P = f3(0.f), n = f3(0.f), a = f3(0.f);
        if (c) {
            float3 org, dir;
            pass_camera_ray<kMotion>(fa, mo, x, y, p, iteration, org, dir);
            P = madd3(org, dir, depth);
            if (ca.normal || ca.albedo) collision_surface(fa, ca, org, dir, P, n, a);
        }
        const float cs = c ? 1.0f : 0.0f;
        if (iteration == 0) { mp = make_float4(P.x, P.y, P.z, cs); mn = n; ma = a; }
        else if (iteration < kp.max_interactions) {
            const float k = (float)(iteration + 1);
            mp.x = mp.x + (P.x - mp.x) / k; mp.y = mp.y + (P.y - mp.y) / k; mp.z = mp.z + (P.z - mp.z) / k; mp.w = mp.w + (cs - mp.w) / k;
            mn.x = mn.x + (n.x - mn.x) / k; mn.y = mn.y + (n.y - mn.y) / k; mn.z = mn.z + (n.z - mn.z) / k;
            ma.x = ma.x + (a.x - ma.x) / k; ma.y = ma.y + (a.y - ma.y) / k; ma.z = ma.z + (a.z - ma.z) / k;
        }
    }
    if (ca.position) ca.position[lp] = mp;
    if (ca.normal) ca.normal[lp] = mn;
    if (ca.albedo) ca.albedo[lp] = ma;
}

__global__ void __launch_bounds__(256)
k_collision_aovs(const FrameArgs fa, const CollisionAovs ca, const int n_passes, const int sampled)
{ frame_pixel(fa.geom, [&](uint32_t lp, int lr, int y) { collision_aovs_pixel<false>(fa, ca, nullptr, n_passes, sampled, lp, lr, y); }); }

__global__ void __launch_bounds__(256)
k_collision_aovs_region(const FrameArgs fa, const CollisionAovs ca, const int n_passes, const int sampled, const RenderRegion rg)
{ region_pixel(fa.geom, rg, [&](uint32_t lp, int lr, int y) { collision_aovs_pixel<false>(fa, ca, nullptr, n_passes, sampled, lp, lr, y); }); }

__global__ void __launch_bounds__(128)
k_collision_aovs_adaptive(const FrameArgs fa, const CollisionAovs ca, const int n_passes, const AdaptArgs ad)
{ adaptive_pixel(fa.geom, ad, [&](uint32_t lp, int lr, int y) { collision_aovs_pixel<false>(fa, ca, nullptr, n_passes, 1, lp, lr, y); }); }

__global__ void __launch_bounds__(256)
k_collision_aovs_motion(const FrameArgs fa, const CollisionAovs ca, const int n_passes, const int sampled, const CameraMotion mo)
{ frame_pixel(fa.geom, [&](uint32_t lp, int lr, int y) { collision_aovs_pixel<true>(fa, ca, &mo, n_passes, sampled, lp, lr, y); }); }

__global__ void __launch_bounds__(256)
k_collision_aovs_region_motion(const FrameArgs fa, const CollisionAovs ca, const int n_passes, const int sampled, const RenderRegion rg,
                               const CameraMotion mo)
{ region_pixel(fa.geom, rg, [&](uint32_t lp, int lr, int y) { collision_aovs_pixel<true>(fa, ca, &mo, n_passes, sampled, lp, lr, y); }); }

__global__ void __launch_bounds__(128)
k_collision_aovs_adaptive_motion(const FrameArgs fa, const CollisionAovs ca, const int n_passes, const AdaptArgs ad, const CameraMotion mo)
{ adaptive_pixel(fa.geom, ad, [&](uint32_t lp, int lr, int y) { collision_aovs_pixel<true>(fa, ca, &mo, n_passes, 1, lp, lr, y); }); }

// =====================================================================================================
// k_cryptomatte: per-pixel instance coverage counted by id; k_cryptomatte_rank: the ranks (DESIGN.md section 8s)
// =====================================================================================================
// A table of up to kCryptoRegEntries entries is kept in registers over the chunk (the loops over it are unrolled, so it never goes to local
// memory); a larger one is searched and counted in its state rows, which a warp reads coalesced and L1 keeps.
constexpr int kCryptoRegEntries = 8;

// One pixel over the chunk's passes.  Entries fill in first-seen order and are never emptied, so the entries with count > 0 are a prefix of
// the table (`used` of them) in every state the kernels write: the search for an id ends at the first empty entry, which is the one a new
// id takes.  The id plane is read only where c holds, where the trace kernel wrote it.
template <bool kRegs>
__device__ __forceinline__ void cryptomatte_pixel(const FrameArgs& fa, const Cryptomatte& cm, const int n_passes, const int sampled, const uint32_t lp)
{
    const vpt_kernel_params& kp = fa.kp;
    const uint32_t it0 = kp.iteration;
    if (it0 >= kp.max_interactions) return;                       // accum's gate: no pass of the chunk changes the state
    const uint32_t left = kp.max_interactions - it0;
    const int n_upd = (uint32_t)n_passes < left ? n_passes : (int)left;
    const size_t n = (size_t)fa.geom.n_local;
    uint32_t* st = cm.state + lp;                                  // plane k of the pixel at st[k * n]
    const int cap = cm.cap;
    const bool clear = it0 == 0;                                   // iteration 0 assigns: the pixel starts empty
    uint32_t count_n = clear ? 0u : st[0];
    uint32_t overflow = clear ? 0u : st[n];
    const bool records = sampled && !(fa.miss_mask && fa.miss_mask[lp]);
    const bool compact = !fa.planeB;
    if constexpr (kRegs) {
        uint32_t ids[kCryptoRegEntries], counts[kCryptoRegEntries];
        int used = 0;
#pragma unroll
        for (int j = 0; j < kCryptoRegEntries; ++j) {
            ids[j] = 0u; counts[j] = 0u;
            if (!clear && j < cap) { ids[j] = st[(size_t)(2 + 2 * j) * n]; counts[j] = st[(size_t)(3 + 2 * j) * n]; }
            if (j == used && counts[j] != 0u) used = j + 1;
        }
        for (int p = 0; p < n_upd; ++p) {
            ++count_n;
            if (!(record_depth(fa, p, lp, records, compact) > 0.0f)) continue;
            const uint32_t id = cm.id[(size_t)p * n + lp];
            bool found = false;
#pragma unroll
            for (int j = 0; j < kCryptoRegEntries; ++j)
                if (j < used && ids[j] == id) { ++counts[j]; found = true; }
            if (found) continue;
            if (used < cap) {
#pragma unroll
                for (int j = 0; j < kCryptoRegEntries; ++j)
                    if (j == used) { ids[j] = id; counts[j] = 1u; }
                ++used;
            } else {
                ++overflow;
            }
        }
#pragma unroll
        for (int j = 0; j < kCryptoRegEntries; ++j)
            if (j < cap && (clear || j < used)) { st[(size_t)(2 + 2 * j) * n] = ids[j]; st[(size_t)(3 + 2 * j) * n] = counts[j]; }
    } else {
        int used = 0;
        if (clear) {
            for (int j = 0; j < cap; ++j) { st[(size_t)(2 + 2 * j) * n] = 0u; st[(size_t)(3 + 2 * j) * n] = 0u; }
        } else {
            while (used < cap && st[(size_t)(3 + 2 * used) * n] != 0u) ++used;
        }
        for (int p = 0; p < n_upd; ++p) {
            ++count_n;
            if (!(record_depth(fa, p, lp, records, compact) > 0.0f)) continue;
            const uint32_t id = cm.id[(size_t)p * n + lp];
            int j = 0;
            while (j < used && st[(size_t)(2 + 2 * j) * n] != id) ++j;
            if (j < used) {
                st[(size_t)(3 + 2 * j) * n] += 1u;
            } else if (used < cap) {
                st[(size_t)(2 + 2 * used) * n] = id; st[(size_t)(3 + 2 * used) * n] = 1u;
                ++used;
            } else {
                ++overflow;
            }
        }
    }
    st[0] = count_n;
    st[n] = overflow;
}

template <bool kRegs>
__global__ void __launch_bounds__(256)
k_cryptomatte(const FrameArgs fa, const Cryptomatte cm, const int n_passes, const int sampled)
{ frame_pixel(fa.geom, [&](uint32_t lp, int, int) { cryptomatte_pixel<kRegs>(fa, cm, n_passes, sampled, lp); }); }

template <bool kRegs>
__global__ void __launch_bounds__(256)
k_cryptomatte_region(const FrameArgs fa, const Cryptomatte cm, const int n_passes, const int sampled, const RenderRegion rg)
{ region_pixel(fa.geom, rg, [&](uint32_t lp, int, int) { cryptomatte_pixel<kRegs>(fa, cm, n_passes, sampled, lp); }); }

template <bool kRegs>
__global__ void __launch_bounds__(128)
k_cryptomatte_adaptive(const FrameArgs fa, const Cryptomatte cm, const int n_passes, const AdaptArgs ad)
{ adaptive_pixel(fa.geom, ad, [&](uint32_t lp, int, int) { cryptomatte_pixel<kRegs>(fa, cm, n_passes, 1, lp); }); }

// One thread per pixel.  The non-empty entries are copied to the thread's own arrays; each entry's rank is the number of non-empty entries
// ahead of it (count greater, or equal count and smaller id: the sphere's id is the largest uint32, so it comes last among equals).
__global__ void __launch_bounds__(256)
k_cryptomatte_rank(const CryptoRank a)
{
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n_px) return;
    const size_t n_px = (size_t)a.n_px;
    const uint32_t n = a.state[i];
    uint32_t ids[kCryptoMaxEntries], counts[kCryptoMaxEntries];
    int m = 0;
    if (n != 0u)
        for (int j = 0; j < a.cap; ++j) {
            const uint32_t c = a.state[(size_t)(3 + 2 * j) * n_px + i];
            if (c != 0u) { ids[m] = a.state[(size_t)(2 + 2 * j) * n_px + i]; counts[m] = c; ++m; }
        }
    const float fn = (float)n;
    for (int k = 0; k < m; ++k) {
        int r = 0;
        for (int q = 0; q < m; ++q) r += (counts[q] > counts[k] || (counts[q] == counts[k] && ids[q] < ids[k])) ? 1 : 0;
        if (r >= a.n_ranks) continue;
        const uint32_t id = ids[k];
        const float idf = id == kMatteSphereId ? a.sphere_id : id < a.n_instances ? __ldg(a.id_of_instance + id) : 0.0f;
        a.out[((size_t)(r >> 1) * n_px + i) * 2 + (r & 1)] = make_float2(idf, __fdiv_rn((float)counts[k], fn));
    }
    for (int r = m; r < a.n_ranks; ++r) a.out[((size_t)(r >> 1) * n_px + i) * 2 + (r & 1)] = make_float2(0.0f, 0.0f);
    if (a.out_overflow) a.out_overflow[i] = n == 0u ? 0.0f : __fdiv_rn((float)a.state[n_px + i], fn);
}

// Convergence test, one block of 128 per active tile: an active pixel stops when the largest err over its 3x3 neighbourhood (global rows,
// clipped at the frame edge; a stopped neighbour counts with the last err it had) is strictly below the threshold.  A neighbour row this
// rank owns is read from ad.stat, a row of another rank from `halo` (the local exchange block's full-frame err plane, which k_adapt_halo of
// every rank filled before the barrier ahead of this launch).  One rank owns every row: the neighbour set is the local one.  A tile with a
// pixel still active is appended to the next list (one atomic per tile).  A NaN err counts as +Inf (fmaxf alone would drop it): such a
// pixel and its neighbours never stop.
// kRegion (k_adapt_region): the neighbourhood is clipped at R's edge instead, so the rule is the one above applied to R as if R were the frame.
template <bool kRegion>
__device__ __forceinline__ void adapt_body(const FrameGeom& g, const AdaptArgs& ad, const float* __restrict__ halo, const RenderRegion* rg)
{
    const int tile = (int)__ldg(ad.tiles + blockIdx.x);
    const TilePixel t = tile_pixel(g, tile);
    const int ylo = kRegion ? rg->y0 : 0, yhi = kRegion ? rg->y1 : g.height;
    const int xlo = kRegion ? rg->x0 : 0, xhi = kRegion ? rg->x1 : g.width;
    bool active = false;
    if (t.inside) {
        const size_t lp = (size_t)t.lr * g.width + t.x;
        if (!ad.stopped[lp]) {
            float worst = 0.0f;
            const int y = g.n_ranks > 1 ? global_row(g, t.lr) : t.lr;
            for (int dy = -1; dy <= 1; ++dy) {
                const int gy = y + dy;
                if (gy < ylo || gy >= yhi) continue;
                int r = gy; bool own = true;                           // r: local row of gy when this rank owns it
                if (g.n_ranks > 1) {
                    const int s = gy / g.stripe_h;
                    own = s % g.n_ranks == g.rank;
                    r = (s / g.n_ranks) * g.stripe_h + (gy - s * g.stripe_h);
                }
                for (int dx = -1; dx <= 1; ++dx) {
                    const int c = t.x + dx;
                    if (c < xlo || c >= xhi) continue;
                    const float e = own ? ad.stat[(size_t)r * g.width + c].w : halo[(size_t)gy * g.width + c];
                    worst = fmaxf(worst, isnan(e) ? INFINITY : e);
                }
            }
            if (worst < ad.threshold) ad.stopped[lp] = 1;
            else active = true;
        }
    }
    if (__syncthreads_or(active) && threadIdx.x == 0) ad.next_tiles[atomicAdd(ad.next_count, 1u)] = (unsigned)tile;
}

__global__ void __launch_bounds__(128)
k_adapt(const FrameGeom g, const AdaptArgs ad, const float* __restrict__ halo) { adapt_body<false>(g, ad, halo, nullptr); }

__global__ void __launch_bounds__(128)
k_adapt_region(const FrameGeom g, const AdaptArgs ad, const RenderRegion rg) { adapt_body<true>(g, ad, nullptr, &rg); }

// vpt_debug_adapt_rule: the passes [p0, p0 + n_passes) of caller-given samples (float3 [pass][pixel], each as it enters the running mean)
// through the pixel's Welford state, over the active tiles as k_resolve_adaptive visits them, and the same stores at the end of the chunk
__global__ void __launch_bounds__(128)
k_debug_adapt_pass(const FrameGeom g, const AdaptArgs ad, const float3* __restrict__ samples, const int p0, const int n_passes)
{
    const TilePixel t = tile_pixel(g, (int)__ldg(ad.tiles + blockIdx.x));
    if (!t.inside) return;
    const uint32_t lp = (uint32_t)t.lr * (uint32_t)g.width + (uint32_t)t.x;
    if (ad.stopped[lp]) return;
    float wn = 0.f, wmean = 0.f, wm2 = 0.f;
    if (p0 > 0) { const float4 st = ad.stat[lp]; wn = st.x; wmean = st.y; wm2 = st.z; }
    for (int p = 0; p < n_passes; ++p) adapt_welford(wn, wmean, wm2, samples[(size_t)(p0 + p) * g.n_local + lp]);
    const float err = adapt_err(wn, wmean, wm2);
    ad.stat[lp] = make_float4(wn, wmean, wm2, err);
    ad.pass_count[lp] = (unsigned)(p0 + n_passes);
    if (ad.rel_error) ad.rel_error[lp] = err;
}

__global__ void k_adapt_init(uint8_t* stopped, unsigned* tiles, int n_local, int n_tiles)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < max(n_local, n_tiles); i += gridDim.x * blockDim.x) {
        if (i < n_local) stopped[i] = 0;
        if (i < n_tiles) tiles[i] = (unsigned)i;
    }
}

// start of an adaptive region frame: the tile list is R's tile rectangle, and every local pixel outside R is stopped -- it never samples
// and never writes, so its buffers, pass count and error keep what they held
__global__ void k_adapt_init_region(const FrameGeom g, uint8_t* stopped, unsigned* tiles, const RenderRegion rg)
{
    const int tiles_x = (g.width + 31) / 32, w = rg.tx1 - rg.tx0, n_tiles = w * (rg.ty1 - rg.ty0);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < max(g.n_local, n_tiles); i += gridDim.x * blockDim.x) {
        if (i < g.n_local) {
            const int lr = i / g.width, x = i - lr * g.width;
            stopped[i] = (x >= rg.x0 && x < rg.x1 && lr >= rg.lr0 && lr < rg.lr1) ? 0 : 1;
        }
        if (i < n_tiles) { const int r = i / w; tiles[i] = (unsigned)((rg.ty0 + r) * tiles_x + rg.tx0 + (i - r * w)); }
    }
}

// ---- sharded adaptive frames (peer-memory exchange) ---------------------------------------------------------------------------------
// Halo, one block of 128 per active tile, after the resolve of a test chunk: a pixel that has not stopped and whose global row has a
// neighbour row of another rank (first / last row of its stripe, inside the frame) stores its err at its global position in every rank's
// err plane.  A stopped pixel's last store stays there, which is what the rule reads for a stopped neighbour.
__global__ void __launch_bounds__(128)
k_adapt_halo(const FrameGeom g, const AdaptArgs ad, const AdaptPeers pp)
{
    const TilePixel t = tile_pixel(g, (int)__ldg(ad.tiles + blockIdx.x));
    if (!t.inside || g.n_ranks < 2) return;
    const int y = global_row(g, t.lr);
    const int off = y % g.stripe_h;
    if (!((off == 0 && y > 0) || (off == g.stripe_h - 1 && y + 1 < g.height))) return;
    const size_t lp = (size_t)t.lr * g.width + t.x;
    if (ad.stopped[lp]) return;
    const float e = ad.stat[lp].w;
    const size_t gp = (size_t)y * g.width + t.x;
    #pragma unroll
    for (int p = 0; p < kMaxPeers; ++p) if (p < pp.n) pp.err[p][gp] = e;
}

// Count publish (lane p -> rank p's block) and the snapshot of the error word taken before the count barrier.
__global__ void k_adapt_count_publish(const AdaptPeers pp, int rank, const unsigned* next_count, const unsigned long long* err_word, unsigned* out)
{
    const int p = threadIdx.x;
    if (p == 0) out[2] = (unsigned)*reinterpret_cast<const volatile unsigned long long*>(err_word);
    if (p < pp.n) pp.tiles[p][rank] = *next_count;
}

__global__ void k_adapt_tally(const unsigned* slots, int n, const unsigned long long* err_word, unsigned* out, int at)
{
    if (threadIdx.x != 0) return;
    if (n > 0) {
        unsigned s = 0;
        for (int p = 0; p < n; ++p) s += reinterpret_cast<const volatile unsigned*>(slots)[p];   // stored by the peers before their flag
        out[1] = s;
    }
    out[at] = (unsigned)*reinterpret_cast<const volatile unsigned long long*>(err_word);
}

// Final publish, one thread per local pixel: the finished pixel at its global position in every rank's planes.
__global__ void __launch_bounds__(256)
k_adapt_publish(const FrameGeom g, const float3* __restrict__ accum, const unsigned* __restrict__ display, unsigned* pass_count, float* rel_error,
                const float4* __restrict__ stat, const AdaptPeers pp)
{
    const uint32_t lp = blockIdx.x * blockDim.x + threadIdx.x;
    if (lp >= (uint32_t)g.n_local) return;
    const int lr = lp / g.width;
    const int y = global_row(g, lr);
    if (y >= g.height) { pass_count[lp] = 0u; if (rel_error) rel_error[lp] = 0.0f; return; }
    const size_t gp = (size_t)y * g.width + (lp - (uint32_t)lr * (uint32_t)g.width);
    const float3 a = accum[lp];
    const unsigned n = pass_count[lp];
    const float e = stat[lp].w;
    const unsigned d = pp.display[0] ? display[lp] : 0u;
    #pragma unroll
    for (int p = 0; p < kMaxPeers; ++p) if (p < pp.n) {
        float* q = pp.accum[p] + 3 * gp; q[0] = a.x; q[1] = a.y; q[2] = a.z;
        if (pp.display[p]) pp.display[p][gp] = d;
        pp.count[p][gp] = n; pp.err[p][gp] = e;
    }
}

// Exchange layers, one thread per pixel of the rectangle rg (the whole local frame, or R's pixels on this rank), row by row as
// k_resolve_region: depth and the active compositing layers at the pixel's global position in every rank's planes, as k_adapt_publish
// does for accum.  A copy behind the resolve, so no resolve kernel's parameter block grows.
__global__ void __launch_bounds__(256)
k_layers_publish(const FrameGeom g, const RenderRegion rg, const LayerSources src, const LayerPlanes dst)
{
    const uint32_t w = (uint32_t)(rg.x1 - rg.x0);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= w * (uint32_t)(rg.lr1 - rg.lr0)) return;
    const uint32_t r = i / w;
    const int lr = rg.lr0 + (int)r, x = rg.x0 + (int)(i - r * w);
    const int y = global_row(g, lr);
    if (y >= g.height) return;                                    // padding row
    const size_t lp = (size_t)lr * g.width + x, gp = (size_t)y * g.width + x;
    #pragma unroll
    for (int l = 0; l < kExchangeLayers; ++l) {
        if (!src.src[l] || !dst.plane[l][0]) continue;             // not active here / not exported (then on no rank: import checks the masks)
        if (l < XL_VOLUME) {
            const float v = src.src[l][lp];
            #pragma unroll
            for (int p = 0; p < kMaxPeers; ++p) if (p < dst.n) dst.plane[l][p][gp] = v;
        } else {
            const float* s = src.src[l] + 3 * lp;
            const float a = s[0], b = s[1], c = s[2];
            #pragma unroll
            for (int p = 0; p < kMaxPeers; ++p) if (p < dst.n) { float* q = dst.plane[l][p] + 3 * gp; q[0] = a; q[1] = b; q[2] = c; }
        }
    }
}

// Binned exchange layers, one thread per (bin k = blockIdx.y, pixel of the rectangle rg), pixels row by row as k_layers_publish walks
// them: bin k of the pixel as one float4 at its global position in every rank's [K][H][W] array.  Adjacent threads take adjacent x, so
// the load and each peer store are coalesced 16-byte accesses.  A copy of its own rather than wider deep / matte resolve kernels: their
// parameter blocks stay as they are.
__global__ void __launch_bounds__(256)
k_binned_publish(const FrameGeom g, const RenderRegion rg, const float4* __restrict__ src, const BinnedPlanes dst)
{
    const uint32_t w = (uint32_t)(rg.x1 - rg.x0);
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= w * (uint32_t)(rg.lr1 - rg.lr0)) return;
    const uint32_t r = i / w;
    const int lr = rg.lr0 + (int)r, x = rg.x0 + (int)(i - r * w);
    const int y = global_row(g, lr);
    if (y >= g.height) return;                                    // padding row
    const size_t k = blockIdx.y;
    const float4 v = src[k * (size_t)g.n_local + (size_t)lr * g.width + x];
    const size_t gp = k * ((size_t)g.width * g.height) + (size_t)y * g.width + x;
    #pragma unroll
    for (int p = 0; p < kMaxPeers; ++p) if (p < dst.n) dst.plane[p][gp] = v;
}

__global__ void k_peer_signal(PeerFlagPtrs fl, int n, int rank, int which, unsigned long long epoch)
{
    const int p = threadIdx.x;
    if (p >= n) return;
    __threadfence_system();                                    // everything this stream stored before (peer frames included) ...
    unsigned long long* slot = fl.p[p] + which * kPeerFlagStride + rank;
    asm volatile("st.release.sys.global.u64 [%0], %1;" :: "l"(slot), "l"(epoch) : "memory");   // ... is visible before the flag
}

__global__ void k_peer_wait(unsigned long long* local, int n, int which, unsigned long long epoch)
{
    const int p = threadIdx.x;
    if (p >= n) return;
    const unsigned long long* slot = local + which * kPeerFlagStride + p;
    unsigned long long t0 = 0; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    for (;;) {
        unsigned long long v; asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(slot) : "memory");
        if (v >= epoch) break;
        unsigned long long t1; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        if (t1 - t0 > 10000000000ull) { atomicAdd(local + 2 * kPeerFlagStride, 1ull); break; }     // 10 s: a rank is gone -- report, do not hang the GPU
        __nanosleep(200);
    }
}

// =====================================================================================================
// k_bn_advance: blue-noise buffer += golden ratio (mod 1), `n` passes worth (:2319-2325)
// =====================================================================================================
// Per-chunk jitter table: table[p][i] = (x, y) of blue-noise entry i after p advances, p = 0..np-1; the buffer
// itself is left advanced by `np` passes.  One launch replaces the per-thread replay in k_generate.
// `limit` = min(W*H, 65536): the reference advances entry idx = y*W + x from the thread of pixel (x, y), so a frame of fewer than
// 65536 pixels leaves the entries beyond W*H untouched (they are still READ as jitter through (y % 256) * 256 + x % 256).
__global__ void k_bn_prepare(float3* bn, float2* table, int np, int limit, unsigned* queue_counters)
{
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx == 0 && queue_counters) { queue_counters[0] = 0u; queue_counters[1] = 0u; }   // first kernel of a round: also resets the ray queue (count, head)
    if (idx >= 256 * 256) return;
    float3 val = bn[idx];
    if (idx >= limit) {
        for (int i = 0; i < np; ++i) table[(size_t)i * 65536 + idx] = make_float2(val.x, val.y);
        return;
    }
    for (int i = 0; i < np; ++i) {
        table[(size_t)i * 65536 + idx] = make_float2(val.x, val.y);
        bn_step(val);
    }
    bn[idx] = val;
}

__global__ void k_bn_advance(float3* bn, int n, int limit)
{
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= 256 * 256 || idx >= limit) return;
    float3 val = bn[idx];
    for (int i = 0; i < n; ++i) bn_step(val);
    bn[idx] = val;
}

// gather permutation for the multi-GPU path: rank-contiguous stripes -> full frame
__global__ void k_unpermute(const uint8_t* __restrict__ gathered, uint8_t* __restrict__ full, FrameGeom g, int elem_bytes)
{
    // one thread per (rank, local pixel) element of 4-byte words
    const size_t words_per_px = elem_bytes / 4;
    const size_t total = (size_t)g.n_ranks * g.n_local * words_per_px;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const size_t px = i / words_per_px, w = i - px * words_per_px;
        const int rank = (int)(px / g.n_local);
        const size_t lp = px - (size_t)rank * g.n_local;
        const int lr = (int)(lp / g.width), x = (int)(lp - (size_t)lr * g.width);
        const int s = lr / g.stripe_h;
        const int y = (s * g.n_ranks + rank) * g.stripe_h + (lr - s * g.stripe_h);
        if (y < g.height)
            reinterpret_cast<uint32_t*>(full)[((size_t)y * g.width + x) * words_per_px + w] = reinterpret_cast<const uint32_t*>(gathered)[i];
    }
}

// vpt_debug_camera_rays: every local pixel's b0 at the jitter of the next render call's first pass (k_bn_prepare's table row 0 is the
// blue-noise buffer as it is now), by the projection's own helper
__global__ void k_camera_rays(const vpt_camera cam, const vpt_u2 res, const FrameGeom g, const Projection pj, const float3* __restrict__ bn, float4* out)
{
    const uint32_t lp = blockIdx.x * blockDim.x + threadIdx.x;
    if (lp >= (uint32_t)g.n_local) return;
    const int lr = lp / g.width, x = lp - lr * g.width;
    const int y = global_row(g, lr);
    if (y >= g.height) { out[lp] = make_float4(0.f, 0.f, 0.f, 0.f); return; }
    const float3 j = bn[(y % 256) * 256 + x % 256];
    const float3 b = pj.kind == kProjEquirect ? pano_b0(cam, pj, res, x, y, j.x, j.y) : camera_b0(cam, res, x, y, j.x, j.y);
    out[lp] = make_float4(b.x, b.y, b.z, 0.f);
}

// vpt_debug_motion_cameras: every local pixel's shutter draw at pass `iteration` -- the lens loop and the draw after it, as k_generate_motion
// takes them (the same radical-inverse tables) -- and the camera motion_camera makes of it
__global__ void k_motion_cameras(const vpt_camera cam, const CameraMotion mo, const FrameGeom g, const uint32_t iteration, float* out)
{
    __shared__ float vdc2[101], vdc3[101];
    if (threadIdx.x < 101) {
        { int n = threadIdx.x; float r = 0, denom = 1, inv = 1.f / 2; while (n) { denom *= 2; r = padd(r, __fdividef((float)(n % 2), denom)); n *= inv; } vdc2[threadIdx.x] = r; }
        { int n = threadIdx.x; float r = 0, denom = 1, inv = 1.f / 3; while (n) { denom *= 3; r = padd(r, __fdividef((float)(n % 3), denom)); n *= inv; } vdc3[threadIdx.x] = r; }
    }
    __syncthreads();
    const uint32_t lp = blockIdx.x * blockDim.x + threadIdx.x;
    if (lp >= (uint32_t)g.n_local) return;
    const int lr = lp / g.width, x = lp - lr * g.width;
    const int y = global_row(g, lr);
    float* o = out + (size_t)lp * 20;
    if (y >= g.height) { for (int i = 0; i < 20; ++i) o[i] = 0.f; return; }
    Rng rng; rng.init((uint32_t)y * (uint32_t)g.width + (uint32_t)x, iteration, 0u);
    float px, py;
    do {
        px = pfma(vdc2[int(rng.next() * 100)], 2.0f, -1.0f);
        py = pfma(vdc3[int(rng.next() * 100)], 2.0f, -1.0f);
    } while (pfma(px, px, pmul(py, py)) >= 1.0f);
    const float xi = rng.next();
    const vpt_camera m = motion_camera(cam, mo, xi);
    const vpt_f3 f[6] = { m.origin, m.lower_left_corner, m.horizontal, m.vertical, m.u, m.v };
    o[0] = xi;
    for (int i = 0; i < 6; ++i) { o[1 + 3 * i] = f[i].x; o[2 + 3 * i] = f[i].y; o[3 + 3 * i] = f[i].z; }
    o[19] = 0.f;
}

// vpt_debug_ods_cameras / vpt_debug_camera_rays on an ODS frame: every local pixel's ods_camera at the jitter `bn` holds now (read only).
// rays == 0: origin', lower_left_corner', e, k (8 floats); rays == 1: (camera_b0 of that camera, 0), the ray direction before normalize
__global__ void k_ods_cameras(const vpt_camera cam, const OdsParams od, const vpt_u2 res, const FrameGeom g, const float3* __restrict__ bn,
                              const int rays, float* out)
{
    const uint32_t lp = blockIdx.x * blockDim.x + threadIdx.x;
    if (lp >= (uint32_t)g.n_local) return;
    const int lr = lp / g.width, x = lp - lr * g.width;
    const int y = global_row(g, lr);
    const int n = rays ? 4 : 8;
    float* o = out + (size_t)lp * n;
    if (y >= g.height) { for (int i = 0; i < n; ++i) o[i] = 0.f; return; }
    const float3 j = bn[(y % 256) * 256 + x % 256];
    const OdsCamera c = ods_camera(cam, od, res, x, y, j.x, j.y);
    if (rays) {
        const float3 b = camera_b0(c.cam, res, x, y, j.x, j.y);
        o[0] = b.x; o[1] = b.y; o[2] = b.z; o[3] = 0.f;
        return;
    }
    o[0] = c.cam.origin.x; o[1] = c.cam.origin.y; o[2] = c.cam.origin.z;
    o[3] = c.cam.lower_left_corner.x; o[4] = c.cam.lower_left_corner.y; o[5] = c.cam.lower_left_corner.z;
    o[6] = c.e; o[7] = c.k;
}

// =====================================================================================================
// host-callable launchers
// =====================================================================================================
cudaError_t launch_prepare_scene(const vpt_gpu_vdb* vols, const vpt_octnode* root, SceneTables* out, OctInternal* internal,
                                 uint2* leaf_list, int* leaf_indices, VolumeRec* vrec, int max_volumes, cudaStream_t s)
{
    SceneTables none; memset(&none, 0, sizeof(none));
    k_prepare_scene<<<4, 256, 0, s>>>(vols, root, out, internal, leaf_list, leaf_indices, vrec, max_volumes, none);
    return cudaGetLastError();
}

cudaError_t launch_prepare_volumes(const vpt_gpu_vdb* vols, const SceneTables& hdr, SceneTables* out, VolumeRec* vrec, cudaStream_t s)
{
    const int blocks = hdr.num_volumes > 4096 ? 32 : 4;
    k_prepare_scene<<<blocks, 256, 0, s>>>(vols, nullptr, out, nullptr, nullptr, nullptr, vrec, hdr.num_volumes, hdr);
    return cudaGetLastError();
}

// one block = a run of 32x4 pixel tiles x a run of passes.  Keep >= ~8 waves of blocks (H100 SXM: 132 SMs x 7 resident blocks) so the tail of the
// grid does not idle the SMs when the local frame is small; never fewer than 4 (tile, pass) pairs per block (amortises the table
// staging: one pass per call used to spend half of this kernel on it).
static dim3 generate_grid(FrameArgs& a, long long tiles, int n_passes)
{
    a.n_passes = n_passes;
    int ppb = n_passes;
    while (ppb > 4 && tiles * ((n_passes + ppb - 1) / ppb) < 7392) ppb = (ppb + 1) / 2;
    int tpb = 1;
    while (ppb * tpb < 4 && tiles / (tpb * 2) >= 2112) tpb *= 2;
    a.passes_per_block = ppb; a.tiles_per_block = tpb;
    return dim3((unsigned)((tiles + tpb - 1) / tpb), 1, (unsigned)((n_passes + ppb - 1) / ppb));
}

cudaError_t launch_generate(const FrameArgs& fa, int n_passes, const Projection& pj, const CameraMotion* mo, const OdsParams* od, cudaStream_t s)
{
    FrameArgs a = fa;
    const long long tiles = (long long)((fa.geom.width + 31) / 32) * ((fa.geom.local_rows + 3) / 4);
    const dim3 grid = generate_grid(a, tiles, n_passes);
    if (mo) k_generate_motion<<<grid, 128, 0, s>>>(a, *mo);
    else if (od) k_generate_ods<<<grid, 128, 0, s>>>(a, *od);
    else if (equirect(pj)) k_generate_equirect<<<grid, 128, 0, s>>>(a, pj);
    else k_generate<<<grid, 128, 0, s>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_miss_cull(const FrameArgs& fa, uint8_t* mask, const Projection& pj, cudaStream_t s, const OdsParams* od)
{
    if (fa.geom.n_local <= 0) return cudaSuccess;
    const long long strips = (long long)fa.geom.local_rows * ((fa.geom.width + kCullStrip - 1) / kCullStrip);
    if (od) k_miss_cull_ods<<<(unsigned)((strips + 255) / 256), 256, 0, s>>>(fa, mask, *od);
    else if (equirect(pj)) k_miss_cull_equirect<<<(unsigned)((strips + 255) / 256), 256, 0, s>>>(fa, mask, pj);
    else k_miss_cull<<<(unsigned)((strips + 255) / 256), 256, 0, s>>>(fa, mask);
    return cudaGetLastError();
}

cudaError_t launch_generate_region(const FrameArgs& fa, int n_passes, const RenderRegion& rg, const Projection& pj, const CameraMotion* mo,
                                   const OdsParams* od, cudaStream_t s)
{
    const long long tiles = region_tiles(rg);
    if (tiles <= 0) return cudaSuccess;
    FrameArgs a = fa;
    const dim3 grid = generate_grid(a, tiles, n_passes);
    if (mo) k_generate_region_motion<<<grid, 128, 0, s>>>(a, rg, *mo);
    else if (od) k_generate_region_ods<<<grid, 128, 0, s>>>(a, rg, *od);
    else if (equirect(pj)) k_generate_region_equirect<<<grid, 128, 0, s>>>(a, rg, pj);
    else k_generate_region<<<grid, 128, 0, s>>>(a, rg);
    return cudaGetLastError();
}

cudaError_t launch_miss_cull_region(const FrameArgs& fa, uint8_t* mask, const RenderRegion& rg, const Projection& pj, cudaStream_t s,
                                    const OdsParams* od)
{
    if (rg.lr1 <= rg.lr0) return cudaSuccess;
    const long long strips = (long long)(rg.lr1 - rg.lr0) * ((rg.x1 + kCullStrip - 1) / kCullStrip - rg.x0 / kCullStrip);
    if (od) k_miss_cull_region_ods<<<(unsigned)((strips + 255) / 256), 256, 0, s>>>(fa, mask, rg, *od);
    else if (equirect(pj)) k_miss_cull_region_equirect<<<(unsigned)((strips + 255) / 256), 256, 0, s>>>(fa, mask, rg, pj);
    else k_miss_cull_region<<<(unsigned)((strips + 255) / 256), 256, 0, s>>>(fa, mask, rg);
    return cudaGetLastError();
}

cudaError_t launch_generate_adaptive(const FrameArgs& fa, int n_passes, const AdaptArgs& ad, const Projection& pj, const CameraMotion* mo,
                                     const OdsParams* od, cudaStream_t s)
{
    if (ad.n_tiles <= 0) return cudaSuccess;
    FrameArgs a = fa;
    const dim3 grid = generate_grid(a, ad.n_tiles, n_passes);
    if (mo) k_generate_adaptive_motion<<<grid, 128, 0, s>>>(a, ad, *mo);
    else if (od) k_generate_adaptive_ods<<<grid, 128, 0, s>>>(a, ad, *od);
    else if (equirect(pj)) k_generate_adaptive_equirect<<<grid, 128, 0, s>>>(a, ad, pj);
    else k_generate_adaptive<<<grid, 128, 0, s>>>(a, ad);
    return cudaGetLastError();
}

cudaError_t launch_empty_ahead(SceneTables* scene, int enable, cudaStream_t s)
{
    k_empty_ahead<<<1, 128, 0, s>>>(reinterpret_cast<SceneAlloc*>(scene), enable);
    return cudaGetLastError();
}

static BrickArgs brick_args(const float* pool, const int dims[3])
{
    BrickArgs ba;
    ba.pool = pool; ba.dimx = dims[0]; ba.dimy = dims[1]; ba.dimz = dims[2];
    ba.nbx = (dims[0] + 3) / 4; ba.nby = (dims[1] + 3) / 4; ba.nbz = (dims[2] + 3) / 4;
    return ba;
}

// The trace kernels: f(kernel, block size, dynamic shared memory, the arguments after FrameArgs) for TraceKernel k.  Launch, shared
// memory opt-in, occupancy and preload all go through this list and resolve_kernels below.  (A unary + forms the pointer of an
// instantiation with a pack argument: inside a template, g++ cannot deduce the lambda's parameter from that template-id.)
template <class F>
static cudaError_t trace_kernel(TraceKernel k, const vpt_atmosphere& atm, const LightGroups& lg, const MatteIds& mi, const BrickArgs& ba, F&& f)
{
    switch (k) {
    case TK_LEAN_3_MATTES:           return f(+k_trace<0, true, 3, false, false, MatteIds>, trace_threads(true, 3), trace_smem_bytes(true, 3), NoAtmo{}, mi);
    case TK_LEAN_2_MATTES:           return f(+k_trace<0, true, 2, false, false, MatteIds>, trace_threads(true, 2), trace_smem_bytes(true, 2), NoAtmo{}, mi);
    case TK_GENERIC_3_MATTES:        return f(+k_trace<0, false, 3, false, false, MatteIds>, trace_threads(false, 3), trace_smem_bytes(false, 3), NoAtmo{}, mi);
    case TK_GENERIC_2_MATTES:        return f(+k_trace<0, false, 2, false, false, MatteIds>, trace_threads(false, 2), trace_smem_bytes(false, 2), NoAtmo{}, mi);
    case TK_VOL_3_MATTES:            return f(+k_trace<1, false, 3, false, false, MatteIds>, trace_threads(false, 3), trace_smem_bytes(false, 3), atm, mi);
    case TK_GENERIC_3_GROUPS_MATTES: return f(+k_trace<0, false, 3, false, true, LightGroups, MatteIds>, trace_threads(false, 3), trace_smem_bytes(false, 3), NoAtmo{}, lg, mi);
    case TK_VOL_3_GROUPS_MATTES:     return f(+k_trace<1, false, 3, false, true, LightGroups, MatteIds>, trace_threads(false, 3), trace_smem_bytes(false, 3), atm, lg, mi);
    case TK_GENERIC_3:        return f(k_trace<0, false, 3>, trace_threads(false, 3), trace_smem_bytes(false, 3), NoAtmo{});
    case TK_LEAN_3:           return f(k_trace<0, true, 3>, trace_threads(true, 3), trace_smem_bytes(true, 3), NoAtmo{});
    case TK_VOL_3:            return f(k_trace<1, false, 3>, trace_threads(false, 3), trace_smem_bytes(false, 3), atm);
    case TK_BRICK:            return f(k_trace_brick, kBrickThreads, (size_t)kBrickThreads * kBrickBytes, ba);
    case TK_GENERIC_2:        return f(k_trace<0, false, 2>, trace_threads(false, 2), trace_smem_bytes(false, 2), NoAtmo{});
    case TK_LEAN_2:           return f(k_trace<0, true, 2>, trace_threads(true, 2), trace_smem_bytes(true, 2), NoAtmo{});
    case TK_LEAN_2_CELLS:     return f(k_trace<0, true, 2, true>, trace_threads(true, 2, true), trace_smem_bytes(true, 2, true), NoAtmo{});
    case TK_GENERIC_3_GROUPS: return f(+k_trace<0, false, 3, false, true, LightGroups>, trace_threads(false, 3), trace_smem_bytes(false, 3), NoAtmo{}, lg);
    case TK_VOL_3_GROUPS:     return f(+k_trace<1, false, 3, false, true, LightGroups>, trace_threads(false, 3), trace_smem_bytes(false, 3), atm, lg);
    default:                  return cudaErrorInvalidValue;
    }
}

// The three resolve kernels of key {S, A, G} whose pack `e` ends with the DeepSlices, in the form of resolve_kernels below
template <int S, bool A, bool G, class F, class Sky, class... E>
static cudaError_t resolve_kernels_deep(F&& f, const Sky& sky, const E&... e)
{
    return f(+k_resolve<S, A, G, E...>, +k_resolve_adaptive<S, A, G, E...>, +k_resolve_region<S, A, G, E...>, sky, e...);
}

// The table of resolve_kernels whose pack ends with `dp`: the deep slices (a DeepSlices) or the instance mattes (a Mattes)
template <class F, class Bins>
static cudaError_t resolve_kernels_binned(const ResolveKey& r, const vpt_atmosphere& atm, const AovBuffers& aov, const LightGroups& lg, const Bins& dp,
                                          F&& f)
{
    const NoSky hdri{};
    switch (r.sky * 4 + r.aov * 2 + r.groups) {
    case 0:  return resolve_kernels_deep<0, false, false>(f, hdri, dp);
    case 1:  return resolve_kernels_deep<0, false, true>(f, hdri, lg, dp);
    case 2:  return resolve_kernels_deep<0, true, false>(f, hdri, aov, dp);
    case 3:  return resolve_kernels_deep<0, true, true>(f, hdri, aov, lg, dp);
    case 4:  return resolve_kernels_deep<1, false, false>(f, atm, dp);
    case 5:  return resolve_kernels_deep<1, false, true>(f, atm, lg, dp);
    case 6:  return resolve_kernels_deep<1, true, false>(f, atm, aov, dp);
    case 7:  return resolve_kernels_deep<1, true, true>(f, atm, aov, lg, dp);
    case 8:  return resolve_kernels_deep<2, false, false>(f, atm, dp);
    case 9:  return resolve_kernels_deep<2, false, true>(f, atm, lg, dp);
    case 10: return resolve_kernels_deep<2, true, false>(f, atm, aov, dp);
    case 11: return resolve_kernels_deep<2, true, true>(f, atm, aov, lg, dp);
    default: return cudaErrorInvalidValue;
    }
}

// The resolve kernels: f(k_resolve<S, A, G>, k_resolve_adaptive<S, A, G>, k_resolve_region<S, A, G>, the sky argument, the trailing
// AovBuffers / LightGroups / DeepSlices or Mattes) for key {S, A, G, D, M}, case S * 4 + A * 2 + G of the table without (D, M false), with
// the deep slices (D) or with the instance mattes (M; D false).
template <class F>
static cudaError_t resolve_kernels(const ResolveKey& r, const vpt_atmosphere& atm, const AovBuffers& aov, const LightGroups& lg, const DeepSlices& dp,
                                   const Mattes& mt, F&& f)
{
    const NoSky hdri{};
    if (r.deep) return resolve_kernels_binned(r, atm, aov, lg, dp, f);
    if (r.mattes) return resolve_kernels_binned(r, atm, aov, lg, mt, f);
    switch (r.sky * 4 + r.aov * 2 + r.groups) {
    case 0:  return f(k_resolve<0>, k_resolve_adaptive<0>, k_resolve_region<0>, hdri);
    case 1:  return f(+k_resolve<0, false, true, LightGroups>, +k_resolve_adaptive<0, false, true, LightGroups>, +k_resolve_region<0, false, true, LightGroups>, hdri, lg);
    case 2:  return f(+k_resolve<0, true, false, AovBuffers>, +k_resolve_adaptive<0, true, false, AovBuffers>, +k_resolve_region<0, true, false, AovBuffers>, hdri, aov);
    case 3:  return f(+k_resolve<0, true, true, AovBuffers, LightGroups>, +k_resolve_adaptive<0, true, true, AovBuffers, LightGroups>, +k_resolve_region<0, true, true, AovBuffers, LightGroups>, hdri, aov, lg);
    case 4:  return f(k_resolve<1>, k_resolve_adaptive<1>, k_resolve_region<1>, atm);
    case 5:  return f(+k_resolve<1, false, true, LightGroups>, +k_resolve_adaptive<1, false, true, LightGroups>, +k_resolve_region<1, false, true, LightGroups>, atm, lg);
    case 6:  return f(+k_resolve<1, true, false, AovBuffers>, +k_resolve_adaptive<1, true, false, AovBuffers>, +k_resolve_region<1, true, false, AovBuffers>, atm, aov);
    case 7:  return f(+k_resolve<1, true, true, AovBuffers, LightGroups>, +k_resolve_adaptive<1, true, true, AovBuffers, LightGroups>, +k_resolve_region<1, true, true, AovBuffers, LightGroups>, atm, aov, lg);
    case 8:  return f(k_resolve<2>, k_resolve_adaptive<2>, k_resolve_region<2>, atm);
    case 9:  return f(+k_resolve<2, false, true, LightGroups>, +k_resolve_adaptive<2, false, true, LightGroups>, +k_resolve_region<2, false, true, LightGroups>, atm, lg);
    case 10: return f(+k_resolve<2, true, false, AovBuffers>, +k_resolve_adaptive<2, true, false, AovBuffers>, +k_resolve_region<2, true, false, AovBuffers>, atm, aov);
    case 11: return f(+k_resolve<2, true, true, AovBuffers, LightGroups>, +k_resolve_adaptive<2, true, true, AovBuffers, LightGroups>, +k_resolve_region<2, true, true, AovBuffers, LightGroups>, atm, aov, lg);
    default: return cudaErrorInvalidValue;
    }
}

template <bool A, bool G, class F, class... E>
static cudaError_t resolve_kernels_equirect_deep(F&& f, const NoSky& sky, const E&... e)
{
    return f(+k_resolve_equirect<A, G, E...>, +k_resolve_adaptive_equirect<A, G, E...>, +k_resolve_region_equirect<A, G, E...>, sky, e...);
}

template <class F, class Bins>
static cudaError_t resolve_kernels_equirect_binned(const ResolveKey& r, const AovBuffers& aov, const LightGroups& lg, const Bins& dp, F&& f)
{
    const NoSky hdri{};
    switch (r.aov * 2 + r.groups) {
    case 0:  return resolve_kernels_equirect_deep<false, false>(f, hdri, dp);
    case 1:  return resolve_kernels_equirect_deep<false, true>(f, hdri, lg, dp);
    case 2:  return resolve_kernels_equirect_deep<true, false>(f, hdri, aov, dp);
    case 3:  return resolve_kernels_equirect_deep<true, true>(f, hdri, aov, lg, dp);
    default: return cudaErrorInvalidValue;
    }
}

// The equirectangular resolve kernels of the HDRI frames, in the form of resolve_kernels: f(k_resolve_equirect<A, G>,
// k_resolve_adaptive_equirect<A, G>, k_resolve_region_equirect<A, G>, the sky argument, the trailing AovBuffers / LightGroups / DeepSlices or
// Mattes), case A * 2 + G of the table without, with the deep slices or with the instance mattes.
template <class F>
static cudaError_t resolve_kernels_equirect(const ResolveKey& r, const AovBuffers& aov, const LightGroups& lg, const DeepSlices& dp, const Mattes& mt,
                                            F&& f)
{
    const NoSky hdri{};
    if (r.sky != 0) return cudaErrorInvalidValue;
    if (r.deep) return resolve_kernels_equirect_binned(r, aov, lg, dp, f);
    if (r.mattes) return resolve_kernels_equirect_binned(r, aov, lg, mt, f);
    switch (r.aov * 2 + r.groups) {
    case 0:  return f(k_resolve_equirect<false, false>, k_resolve_adaptive_equirect<false, false>, k_resolve_region_equirect<false, false>, hdri);
    case 1:  return f(+k_resolve_equirect<false, true, LightGroups>, +k_resolve_adaptive_equirect<false, true, LightGroups>, +k_resolve_region_equirect<false, true, LightGroups>, hdri, lg);
    case 2:  return f(+k_resolve_equirect<true, false, AovBuffers>, +k_resolve_adaptive_equirect<true, false, AovBuffers>, +k_resolve_region_equirect<true, false, AovBuffers>, hdri, aov);
    case 3:  return f(+k_resolve_equirect<true, true, AovBuffers, LightGroups>, +k_resolve_adaptive_equirect<true, true, AovBuffers, LightGroups>, +k_resolve_region_equirect<true, true, AovBuffers, LightGroups>, hdri, aov, lg);
    default: return cudaErrorInvalidValue;
    }
}

template <bool A, bool G, class F, class... E>
static cudaError_t resolve_kernels_ods_deep(F&& f, const NoSky& sky, const E&... e)
{
    return f(+k_resolve_ods<A, G, E...>, +k_resolve_adaptive_ods<A, G, E...>, +k_resolve_region_ods<A, G, E...>, sky, e...);
}

template <class F, class Bins>
static cudaError_t resolve_kernels_ods_binned(const ResolveKey& r, const AovBuffers& aov, const LightGroups& lg, const Bins& dp, F&& f)
{
    const NoSky hdri{};
    switch (r.aov * 2 + r.groups) {
    case 0:  return resolve_kernels_ods_deep<false, false>(f, hdri, dp);
    case 1:  return resolve_kernels_ods_deep<false, true>(f, hdri, lg, dp);
    case 2:  return resolve_kernels_ods_deep<true, false>(f, hdri, aov, dp);
    case 3:  return resolve_kernels_ods_deep<true, true>(f, hdri, aov, lg, dp);
    default: return cudaErrorInvalidValue;
    }
}

// The ODS resolve kernels of the HDRI frames, in the form of resolve_kernels_equirect
template <class F>
static cudaError_t resolve_kernels_ods(const ResolveKey& r, const AovBuffers& aov, const LightGroups& lg, const DeepSlices& dp, const Mattes& mt, F&& f)
{
    const NoSky hdri{};
    if (r.sky != 0) return cudaErrorInvalidValue;
    if (r.deep) return resolve_kernels_ods_binned(r, aov, lg, dp, f);
    if (r.mattes) return resolve_kernels_ods_binned(r, aov, lg, mt, f);
    switch (r.aov * 2 + r.groups) {
    case 0:  return f(k_resolve_ods<false, false>, k_resolve_adaptive_ods<false, false>, k_resolve_region_ods<false, false>, hdri);
    case 1:  return f(+k_resolve_ods<false, true, LightGroups>, +k_resolve_adaptive_ods<false, true, LightGroups>, +k_resolve_region_ods<false, true, LightGroups>, hdri, lg);
    case 2:  return f(+k_resolve_ods<true, false, AovBuffers>, +k_resolve_adaptive_ods<true, false, AovBuffers>, +k_resolve_region_ods<true, false, AovBuffers>, hdri, aov);
    case 3:  return f(+k_resolve_ods<true, true, AovBuffers, LightGroups>, +k_resolve_adaptive_ods<true, true, AovBuffers, LightGroups>, +k_resolve_region_ods<true, true, AovBuffers, LightGroups>, hdri, aov, lg);
    default: return cudaErrorInvalidValue;
    }
}

cudaError_t launch_trace(const FrameArgs& fa, TraceKernel k, const vpt_atmosphere& atm, const LightGroups& lg, const MatteIds& mi,
                         const float* brick_pool, const int brick_dims[3], int n_ctas, cudaStream_t s)
{
    return trace_kernel(k, atm, lg, mi, brick_args(brick_pool, brick_dims), [&](auto kernel, int threads, size_t smem, const auto&... args) {
        kernel<<<n_ctas, threads, smem, s>>>(fa, args...);
        return cudaGetLastError();
    });
}

static_assert(sizeof(FrameShared) + sizeof(EmptyAhead) <= kTraceTablesBytes, "k_trace's static shared memory outgrew kTraceTablesBytes");
static_assert(trace_sm_smem_bytes(true, 2) <= kSmemPerSm && trace_sm_smem_bytes(true, 2, true) <= kSmemPerSm && trace_sm_smem_bytes(false, 2) <= kSmemPerSm,
              "trace CTAs do not fit an SM");

// Once per context (= per device): opt the trace kernels into their dynamic shared memory and record how many CTAs of each fit
// on an SM.  The attribute is a per-device property of the function, so this must not be a process-wide static.  The lean kernels at
// 2 rays per lane must fit trace_min_ctas CTAs; under VPT_LEAN2_SHAPE 1 they ask for the least shared-memory carveout that holds them
// (the rest of the 256 KB is L1).
cudaError_t trace_kernels_init(int max_ctas[kTraceKernelsAll])
{
    for (int k = 0; k < kTraceKernelsAll; ++k) {
        const bool lean2 = k == TK_LEAN_2 || k == TK_LEAN_2_MATTES || k == TK_LEAN_2_CELLS, cells = k == TK_LEAN_2_CELLS;
        const cudaError_t e = trace_kernel((TraceKernel)k, {}, {}, {}, {}, [&](auto kernel, int threads, size_t smem, const auto&...) {
            cudaError_t r = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (r == cudaSuccess && lean2 && VPT_LEAN2_SHAPE == 1) r = cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, trace_carveout_percent(true, 2, cells));
            if (r == cudaSuccess) r = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&max_ctas[k], kernel, threads, smem);
            if (r == cudaSuccess && lean2 && max_ctas[k] < trace_min_ctas(true, 2, cells)) r = cudaErrorInvalidConfiguration;
            return r;
        });
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// Under lazy module loading (the CUDA 12 default) the first launch of a kernel loads it, and loading may wait for the device's running
// kernels.  With a peer exchange, a rank's k_peer_wait spins until the other ranks' kernels have run, so a first launch on one rank
// can wait behind that spin until the wait gives up.  The exchange therefore loads every kernel it may issue up front.
cudaError_t exchange_kernels_preload()
{
    auto load = [](auto... kernels) {
        for (const void* f : {(const void*)kernels...}) {
            cudaFuncAttributes a;
            const cudaError_t e = cudaFuncGetAttributes(&a, f);
            if (e != cudaSuccess) return e;
        }
        return cudaSuccess;
    };
    for (int k = 0; k < kTraceKernelsAll; ++k) {
        const cudaError_t e = trace_kernel((TraceKernel)k, {}, {}, {}, {}, [&](auto kernel, int, size_t, const auto&...) { return load(kernel); });
        if (e != cudaSuccess) return e;
    }
    for (int sky = 0; sky < 3; ++sky)
        for (bool aov : {false, true})
            for (bool groups : {false, true})
                for (int bins = 0; bins < 3; ++bins) {                 // none, the deep slices, the instance mattes
                    const ResolveKey key{sky, aov, groups, bins == 1, bins == 2};
                    const cudaError_t e = resolve_kernels(key, {}, {}, {}, {}, {},
                                                          [&](auto fixed, auto adaptive, auto region, const auto&...) { return load(fixed, adaptive, region); });
                    if (e != cudaSuccess) return e;
                    if (sky != 0) continue;
                    const cudaError_t ep = resolve_kernels_equirect(key, {}, {}, {}, {},
                                                                    [&](auto fixed, auto adaptive, auto region, const auto&...) { return load(fixed, adaptive, region); });
                    if (ep != cudaSuccess) return ep;
                    const cudaError_t eo = resolve_kernels_ods(key, {}, {}, {}, {},
                                                               [&](auto fixed, auto adaptive, auto region, const auto&...) { return load(fixed, adaptive, region); });
                    if (eo != cudaSuccess) return eo;
                }
    return load(k_prepare_scene, k_bn_prepare, k_bn_advance, k_miss_cull, k_generate, k_generate_adaptive, k_adapt_init, k_adapt, k_adapt_halo,
                k_adapt_count_publish, k_adapt_tally, k_adapt_publish, k_peer_signal, k_peer_wait, k_generate_region, k_miss_cull_region,
                k_adapt_init_region, k_adapt_region, k_generate_equirect, k_generate_adaptive_equirect, k_generate_region_equirect,
                k_miss_cull_equirect, k_miss_cull_region_equirect, k_layers_publish, k_generate_motion, k_generate_adaptive_motion,
                k_generate_region_motion, k_generate_ods, k_generate_adaptive_ods, k_generate_region_ods, k_miss_cull_ods, k_miss_cull_region_ods,
                k_binned_publish, k_empty_ahead, k_motion_vectors, k_motion_vectors_region, k_motion_vectors_adaptive,
                k_motion_vectors_motion, k_motion_vectors_region_motion, k_motion_vectors_adaptive_motion, k_collision_aovs,
                k_collision_aovs_region, k_collision_aovs_adaptive, k_collision_aovs_motion, k_collision_aovs_region_motion,
                k_collision_aovs_adaptive_motion, k_cryptomatte<true>, k_cryptomatte<false>, k_cryptomatte_region<true>,
                k_cryptomatte_region<false>, k_cryptomatte_adaptive<true>, k_cryptomatte_adaptive<false>, k_cryptomatte_rank);
}

cudaError_t launch_sampler_compare(unsigned long long tex, const float* pool, const int dims[3], int n, unsigned seed, double* d_out12, cudaStream_t s)
{
    k_sampler_compare<<<592, 256, 0, s>>>((cudaTextureObject_t)tex, brick_args(pool, dims), n, seed, d_out12);
    return cudaGetLastError();
}

cudaError_t launch_software_sample(const float* pool, const float4* cells, const int dims[3], const float* d_uvw, int n, float* d_out2, cudaStream_t s)
{
    const int per_block = kSampleThreads * kSamplePointsPerLane;
    k_software_sample<<<(n + per_block - 1) / per_block, kSampleThreads, (size_t)kSampleThreads * kBrickBytes, s>>>(brick_args(pool, dims), cells, d_uvw, n, d_out2);
    return cudaGetLastError();
}

static cudaError_t resolve_launch(const FrameArgs& fa, const ResolveKey& key, const vpt_atmosphere& atm, int n_passes, int sampled, int write_display,
                                  const PeerFrames* peers, const AovBuffers& aov, const LightGroups& lg, const DeepSlices& dp, const Mattes& mt,
                                  const Projection& pj, const OdsParams* od, cudaStream_t s)
{
    const int threads = 256;
    const int blocks = (fa.geom.n_local + threads - 1) / threads;
    const PeerFrames pf = peers ? *peers : PeerFrames{};
    if (od && key.sky == 0)
        return resolve_kernels_ods(key, aov, lg, dp, mt, [&](auto kernel, auto, auto, const auto& sky, const auto&... ext) {
            kernel<<<blocks, threads, 0, s>>>(fa, sky, n_passes, sampled, write_display, pf, *od, ext...);
            return cudaGetLastError();
        });
    if (equirect(pj) && key.sky == 0)
        return resolve_kernels_equirect(key, aov, lg, dp, mt, [&](auto kernel, auto, auto, const auto& sky, const auto&... ext) {
            kernel<<<blocks, threads, 0, s>>>(fa, sky, n_passes, sampled, write_display, pf, pj, ext...);
            return cudaGetLastError();
        });
    // (tried for frames of less than two waves of blocks -- multi-GPU shards: fetching the records of four passes at once before the
    // order-dependent running mean; slower there too)
    return resolve_kernels(key, atm, aov, lg, dp, mt, [&](auto kernel, auto, auto, const auto& sky, const auto&... ext) {
        kernel<<<blocks, threads, 0, s>>>(fa, sky, n_passes, sampled, write_display, pf, ext...);
        return cudaGetLastError();
    });
}

static cudaError_t resolve_region_launch(const FrameArgs& fa, const ResolveKey& key, const vpt_atmosphere& atm, int n_passes, int sampled,
                                         int write_display, const PeerFrames* peers, const AovBuffers& aov, const LightGroups& lg, const DeepSlices& dp,
                                         const Mattes& mt, const RenderRegion& rg, const Projection& pj, const OdsParams* od, cudaStream_t s)
{
    const long long n = region_pixels(rg);
    if (n <= 0) return cudaSuccess;
    const int threads = 256;
    const PeerFrames pf = peers ? *peers : PeerFrames{};
    if (od && key.sky == 0)
        return resolve_kernels_ods(key, aov, lg, dp, mt, [&](auto, auto, auto kernel, const auto& sky, const auto&... ext) {
            kernel<<<(unsigned)((n + threads - 1) / threads), threads, 0, s>>>(fa, sky, n_passes, sampled, write_display, pf, rg, *od, ext...);
            return cudaGetLastError();
        });
    if (equirect(pj) && key.sky == 0)
        return resolve_kernels_equirect(key, aov, lg, dp, mt, [&](auto, auto, auto kernel, const auto& sky, const auto&... ext) {
            kernel<<<(unsigned)((n + threads - 1) / threads), threads, 0, s>>>(fa, sky, n_passes, sampled, write_display, pf, rg, pj, ext...);
            return cudaGetLastError();
        });
    return resolve_kernels(key, atm, aov, lg, dp, mt, [&](auto, auto, auto kernel, const auto& sky, const auto&... ext) {
        kernel<<<(unsigned)((n + threads - 1) / threads), threads, 0, s>>>(fa, sky, n_passes, sampled, write_display, pf, rg, ext...);
        return cudaGetLastError();
    });
}

static cudaError_t resolve_adaptive_launch(const FrameArgs& fa, const ResolveKey& key, const vpt_atmosphere& atm, int n_passes, const AdaptArgs& ad,
                                           const AovBuffers& aov, const LightGroups& lg, const DeepSlices& dp, const Mattes& mt,
                                           const Projection& pj, const OdsParams* od, cudaStream_t s)
{
    if (ad.n_tiles <= 0) return cudaSuccess;
    if (od && key.sky == 0)
        return resolve_kernels_ods(key, aov, lg, dp, mt, [&](auto, auto kernel, auto, const auto& sky, const auto&... ext) {
            kernel<<<ad.n_tiles, 128, 0, s>>>(fa, sky, n_passes, ad, *od, ext...);
            return cudaGetLastError();
        });
    if (equirect(pj) && key.sky == 0)
        return resolve_kernels_equirect(key, aov, lg, dp, mt, [&](auto, auto kernel, auto, const auto& sky, const auto&... ext) {
            kernel<<<ad.n_tiles, 128, 0, s>>>(fa, sky, n_passes, ad, pj, ext...);
            return cudaGetLastError();
        });
    return resolve_kernels(key, atm, aov, lg, dp, mt, [&](auto, auto kernel, auto, const auto& sky, const auto&... ext) {
        kernel<<<ad.n_tiles, 128, 0, s>>>(fa, sky, n_passes, ad, ext...);
        return cudaGetLastError();
    });
}

// With deep slices (key.deep) a resolve is two launches: the deep instantiation, which keeps the slices only and reads accum and the AOVs
// before they change, then the frame's own kernel, the very one without slices -- so every other output is bit for bit the same.  The
// instance mattes (key.mattes) take one more launch of the same kind, after the deep one.
static ResolveKey only_deep(const ResolveKey& key) { ResolveKey k = key; k.mattes = false; return k; }
static ResolveKey only_mattes(const ResolveKey& key) { ResolveKey k = key; k.deep = false; return k; }
static ResolveKey without_deep(const ResolveKey& key) { ResolveKey k = key; k.deep = false; k.mattes = false; return k; }

cudaError_t launch_resolve(const FrameArgs& fa, const ResolveKey& key, const vpt_atmosphere& atm, int n_passes, int sampled, int write_display,
                           const PeerFrames* peers, const AovBuffers& aov, const LightGroups& lg, const DeepSlices& dp, const Mattes& mt,
                           const Projection& pj, cudaStream_t s, const OdsParams* od)
{
    if (key.deep) {
        const cudaError_t e = resolve_launch(fa, only_deep(key), atm, n_passes, sampled, 0, nullptr, aov, lg, dp, mt, pj, od, s);
        if (e != cudaSuccess) return e;
    }
    if (key.mattes) {
        const cudaError_t e = resolve_launch(fa, only_mattes(key), atm, n_passes, sampled, 0, nullptr, aov, lg, dp, mt, pj, od, s);
        if (e != cudaSuccess) return e;
    }
    return resolve_launch(fa, without_deep(key), atm, n_passes, sampled, write_display, peers, aov, lg, dp, mt, pj, od, s);
}

cudaError_t launch_resolve_region(const FrameArgs& fa, const ResolveKey& key, const vpt_atmosphere& atm, int n_passes, int sampled, int write_display,
                                  const PeerFrames* peers, const AovBuffers& aov, const LightGroups& lg, const DeepSlices& dp, const Mattes& mt,
                                  const RenderRegion& rg, const Projection& pj, cudaStream_t s, const OdsParams* od)
{
    if (key.deep) {
        const cudaError_t e = resolve_region_launch(fa, only_deep(key), atm, n_passes, sampled, 0, nullptr, aov, lg, dp, mt, rg, pj, od, s);
        if (e != cudaSuccess) return e;
    }
    if (key.mattes) {
        const cudaError_t e = resolve_region_launch(fa, only_mattes(key), atm, n_passes, sampled, 0, nullptr, aov, lg, dp, mt, rg, pj, od, s);
        if (e != cudaSuccess) return e;
    }
    return resolve_region_launch(fa, without_deep(key), atm, n_passes, sampled, write_display, peers, aov, lg, dp, mt, rg, pj, od, s);
}

cudaError_t launch_resolve_adaptive(const FrameArgs& fa, const ResolveKey& key, const vpt_atmosphere& atm, int n_passes, const AdaptArgs& ad,
                                    const AovBuffers& aov, const LightGroups& lg, const DeepSlices& dp, const Mattes& mt, const Projection& pj,
                                    cudaStream_t s, const OdsParams* od)
{
    if (key.deep) {
        const cudaError_t e = resolve_adaptive_launch(fa, only_deep(key), atm, n_passes, ad, aov, lg, dp, mt, pj, od, s);
        if (e != cudaSuccess) return e;
    }
    if (key.mattes) {
        const cudaError_t e = resolve_adaptive_launch(fa, only_mattes(key), atm, n_passes, ad, aov, lg, dp, mt, pj, od, s);
        if (e != cudaSuccess) return e;
    }
    return resolve_adaptive_launch(fa, without_deep(key), atm, n_passes, ad, aov, lg, dp, mt, pj, od, s);
}

cudaError_t launch_motion_vectors(const FrameArgs& fa, const MotionVectors& mv, int n_passes, int sampled, const RenderRegion* rg,
                                  const AdaptArgs* ad, const CameraMotion* mo, cudaStream_t s)
{
    if (ad) {
        if (ad->n_tiles <= 0) return cudaSuccess;
        if (mo) k_motion_vectors_adaptive_motion<<<ad->n_tiles, 128, 0, s>>>(fa, mv, n_passes, *ad, *mo);
        else k_motion_vectors_adaptive<<<ad->n_tiles, 128, 0, s>>>(fa, mv, n_passes, *ad);
    } else if (rg) {
        const long long n = region_pixels(*rg);
        if (n <= 0) return cudaSuccess;
        const unsigned blocks = (unsigned)((n + 255) / 256);
        if (mo) k_motion_vectors_region_motion<<<blocks, 256, 0, s>>>(fa, mv, n_passes, sampled, *rg, *mo);
        else k_motion_vectors_region<<<blocks, 256, 0, s>>>(fa, mv, n_passes, sampled, *rg);
    } else {
        if (fa.geom.n_local <= 0) return cudaSuccess;
        const unsigned blocks = (unsigned)((fa.geom.n_local + 255) / 256);
        if (mo) k_motion_vectors_motion<<<blocks, 256, 0, s>>>(fa, mv, n_passes, sampled, *mo);
        else k_motion_vectors<<<blocks, 256, 0, s>>>(fa, mv, n_passes, sampled);
    }
    return cudaGetLastError();
}

cudaError_t launch_collision_aovs(const FrameArgs& fa, const CollisionAovs& ca, int n_passes, int sampled, const RenderRegion* rg,
                                  const AdaptArgs* ad, const CameraMotion* mo, cudaStream_t s)
{
    if (ad) {
        if (ad->n_tiles <= 0) return cudaSuccess;
        if (mo) k_collision_aovs_adaptive_motion<<<ad->n_tiles, 128, 0, s>>>(fa, ca, n_passes, *ad, *mo);
        else k_collision_aovs_adaptive<<<ad->n_tiles, 128, 0, s>>>(fa, ca, n_passes, *ad);
    } else if (rg) {
        const long long n = region_pixels(*rg);
        if (n <= 0) return cudaSuccess;
        const unsigned blocks = (unsigned)((n + 255) / 256);
        if (mo) k_collision_aovs_region_motion<<<blocks, 256, 0, s>>>(fa, ca, n_passes, sampled, *rg, *mo);
        else k_collision_aovs_region<<<blocks, 256, 0, s>>>(fa, ca, n_passes, sampled, *rg);
    } else {
        if (fa.geom.n_local <= 0) return cudaSuccess;
        const unsigned blocks = (unsigned)((fa.geom.n_local + 255) / 256);
        if (mo) k_collision_aovs_motion<<<blocks, 256, 0, s>>>(fa, ca, n_passes, sampled, *mo);
        else k_collision_aovs<<<blocks, 256, 0, s>>>(fa, ca, n_passes, sampled);
    }
    return cudaGetLastError();
}

// the table in registers when it fits there (kCryptoRegEntries), else in the state rows
cudaError_t launch_cryptomatte(const FrameArgs& fa, const Cryptomatte& cm, int n_passes, int sampled, const RenderRegion* rg, const AdaptArgs* ad,
                               cudaStream_t s)
{
    const bool regs = cm.cap <= kCryptoRegEntries;
    if (ad) {
        if (ad->n_tiles <= 0) return cudaSuccess;
        if (regs) k_cryptomatte_adaptive<true><<<ad->n_tiles, 128, 0, s>>>(fa, cm, n_passes, *ad);
        else k_cryptomatte_adaptive<false><<<ad->n_tiles, 128, 0, s>>>(fa, cm, n_passes, *ad);
    } else if (rg) {
        const long long n = region_pixels(*rg);
        if (n <= 0) return cudaSuccess;
        const unsigned blocks = (unsigned)((n + 255) / 256);
        if (regs) k_cryptomatte_region<true><<<blocks, 256, 0, s>>>(fa, cm, n_passes, sampled, *rg);
        else k_cryptomatte_region<false><<<blocks, 256, 0, s>>>(fa, cm, n_passes, sampled, *rg);
    } else {
        if (fa.geom.n_local <= 0) return cudaSuccess;
        const unsigned blocks = (unsigned)((fa.geom.n_local + 255) / 256);
        if (regs) k_cryptomatte<true><<<blocks, 256, 0, s>>>(fa, cm, n_passes, sampled);
        else k_cryptomatte<false><<<blocks, 256, 0, s>>>(fa, cm, n_passes, sampled);
    }
    return cudaGetLastError();
}

cudaError_t launch_cryptomatte_rank(const CryptoRank& a, cudaStream_t s)
{
    if (a.n_px <= 0) return cudaSuccess;
    k_cryptomatte_rank<<<(unsigned)((a.n_px + 255) / 256), 256, 0, s>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_adapt(const FrameGeom& g, const AdaptArgs& ad, const float* halo, cudaStream_t s)
{
    if (ad.n_tiles <= 0) return cudaSuccess;
    k_adapt<<<ad.n_tiles, 128, 0, s>>>(g, ad, halo);
    return cudaGetLastError();
}

cudaError_t launch_adapt_halo(const FrameGeom& g, const AdaptArgs& ad, const AdaptPeers& pp, cudaStream_t s)
{
    if (ad.n_tiles <= 0 || g.n_ranks < 2) return cudaSuccess;
    k_adapt_halo<<<ad.n_tiles, 128, 0, s>>>(g, ad, pp);
    return cudaGetLastError();
}

cudaError_t launch_adapt_count_publish(const AdaptPeers& pp, int rank, const unsigned* next_count, const unsigned long long* err_word,
                                       unsigned* out, cudaStream_t s)
{
    k_adapt_count_publish<<<1, 32, 0, s>>>(pp, rank, next_count, err_word, out);
    return cudaGetLastError();
}

cudaError_t launch_adapt_tally(const unsigned* slots, int n, const unsigned long long* err_word, unsigned* out, int at, cudaStream_t s)
{
    k_adapt_tally<<<1, 32, 0, s>>>(slots, n, err_word, out, at);
    return cudaGetLastError();
}

cudaError_t launch_adapt_publish(const FrameGeom& g, const vpt_kernel_params& kp, const AdaptArgs& ad, const AdaptPeers& pp, cudaStream_t s)
{
    if (g.n_local <= 0) return cudaSuccess;
    k_adapt_publish<<<(g.n_local + 255) / 256, 256, 0, s>>>(g, reinterpret_cast<const float3*>(kp.accum_buffer),
                                                            reinterpret_cast<const unsigned*>(kp.display_buffer), ad.pass_count, ad.rel_error, ad.stat, pp);
    return cudaGetLastError();
}

cudaError_t launch_layers_publish(const FrameGeom& g, const RenderRegion* rg, const LayerSources& src, const LayerPlanes& dst, cudaStream_t s)
{
    RenderRegion all;                                             // the whole local frame
    all.x1 = g.width; all.lr1 = g.local_rows;
    const RenderRegion& r = rg ? *rg : all;
    const long long n = region_pixels(r);
    if (n <= 0 || dst.n <= 0) return cudaSuccess;
    k_layers_publish<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(g, r, src, dst);
    return cudaGetLastError();
}

cudaError_t launch_binned_publish(const FrameGeom& g, const RenderRegion* rg, const float4* src, int n_bins, const BinnedPlanes& dst, cudaStream_t s)
{
    RenderRegion all;                                             // the whole local frame
    all.x1 = g.width; all.lr1 = g.local_rows;
    const RenderRegion& r = rg ? *rg : all;
    const long long n = region_pixels(r);
    if (n <= 0 || n_bins <= 0 || dst.n <= 0 || !src) return cudaSuccess;
    k_binned_publish<<<dim3((unsigned)((n + 255) / 256), (unsigned)n_bins), 256, 0, s>>>(g, r, src, dst);
    return cudaGetLastError();
}

cudaError_t launch_adapt_init(const FrameGeom& g, uint8_t* stopped, unsigned* tiles, int n_tiles, cudaStream_t s)
{
    k_adapt_init<<<1184, 256, 0, s>>>(stopped, tiles, g.n_local, n_tiles);
    return cudaGetLastError();
}

cudaError_t launch_adapt_init_region(const FrameGeom& g, uint8_t* stopped, unsigned* tiles, const RenderRegion& rg, cudaStream_t s)
{
    k_adapt_init_region<<<1184, 256, 0, s>>>(g, stopped, tiles, rg);
    return cudaGetLastError();
}

cudaError_t launch_adapt_region(const FrameGeom& g, const AdaptArgs& ad, const RenderRegion& rg, cudaStream_t s)
{
    if (ad.n_tiles <= 0) return cudaSuccess;
    k_adapt_region<<<ad.n_tiles, 128, 0, s>>>(g, ad, rg);
    return cudaGetLastError();
}

cudaError_t launch_debug_adapt_pass(const FrameGeom& g, const AdaptArgs& ad, const float3* samples, int p0, int n_passes, cudaStream_t s)
{
    if (ad.n_tiles <= 0 || n_passes <= 0) return cudaSuccess;
    k_debug_adapt_pass<<<ad.n_tiles, 128, 0, s>>>(g, ad, samples, p0, n_passes);
    return cudaGetLastError();
}

cudaError_t launch_peer_signal(unsigned long long* const peer_flags[kMaxPeers], int n, int rank, int which, unsigned long long epoch, cudaStream_t s)
{
    PeerFlagPtrs fl; for (int p = 0; p < kMaxPeers; ++p) fl.p[p] = p < n ? peer_flags[p] : nullptr;
    k_peer_signal<<<1, 32, 0, s>>>(fl, n, rank, which, epoch);
    return cudaGetLastError();
}

cudaError_t launch_peer_wait(unsigned long long* local_flags, int n, int which, unsigned long long epoch, cudaStream_t s)
{
    k_peer_wait<<<1, 32, 0, s>>>(local_flags, n, which, epoch);
    return cudaGetLastError();
}

cudaError_t launch_bn_prepare(void* bn, float2* table, int np, int limit, unsigned* queue_counters, cudaStream_t s)
{
    k_bn_prepare<<<256, 256, 0, s>>>(reinterpret_cast<float3*>(bn), table, np, limit, queue_counters);
    return cudaGetLastError();
}

cudaError_t launch_bn_advance(void* bn, int n, int limit, cudaStream_t s)
{
    k_bn_advance<<<256, 256, 0, s>>>(reinterpret_cast<float3*>(bn), n, limit);
    return cudaGetLastError();
}

cudaError_t launch_camera_rays(const vpt_camera& cam, const vpt_u2 res, const FrameGeom& g, const Projection& pj, const void* bn, float4* out,
                               cudaStream_t s)
{
    if (g.n_local <= 0) return cudaSuccess;
    k_camera_rays<<<(g.n_local + 255) / 256, 256, 0, s>>>(cam, res, g, pj, reinterpret_cast<const float3*>(bn), out);
    return cudaGetLastError();
}

cudaError_t launch_motion_cameras(const vpt_camera& cam, const CameraMotion& mo, const FrameGeom& g, uint32_t iteration, float* out, cudaStream_t s)
{
    if (g.n_local <= 0) return cudaSuccess;
    k_motion_cameras<<<(g.n_local + 255) / 256, 256, 0, s>>>(cam, mo, g, iteration, out);
    return cudaGetLastError();
}

cudaError_t launch_ods_cameras(const vpt_camera& cam, const OdsParams& od, const vpt_u2 res, const FrameGeom& g, const void* bn, int rays, float* out,
                               cudaStream_t s)
{
    if (g.n_local <= 0) return cudaSuccess;
    k_ods_cameras<<<(g.n_local + 255) / 256, 256, 0, s>>>(cam, od, res, g, reinterpret_cast<const float3*>(bn), rays, out);
    return cudaGetLastError();
}

cudaError_t launch_unpermute(const void* gathered, void* full, const FrameGeom& g, int elem_bytes, cudaStream_t s)
{
    k_unpermute<<<1184, 256, 0, s>>>(reinterpret_cast<const uint8_t*>(gathered), reinterpret_cast<uint8_t*>(full), g, elem_bytes);
    return cudaGetLastError();
}

} // namespace vpt
