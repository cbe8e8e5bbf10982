// vpt_trace_brick.cuh -- k_trace_brick: the trace stage for volumes that do not fit any cache (BASELINE configs[3], the
// 1024^3 grid: 4 GiB), reading the density from a BRICK POOL in HBM instead of a 3-D texture ("fast mode").
// (included from vpt_kernels.cu inside `namespace vpt`, after vpt_trace.cuh)
//
// Layout (vpt_bricks.cu): 4x4x4-cell bricks stored with their +1 apron as 5x5x5 texels, 512 bytes each, contiguous.
// Every LANE owns one 512-byte slot of shared memory and one mbarrier.  When a look-up leaves the lane's resident brick
// the lane issues ONE bulk asynchronous copy (TMA: cp.async.bulk.shared.global, SASS UBLKCP) of the new brick into its slot
// and waits on its mbarrier's transaction count; the free-flight steps that follow (mean step = one voxel at the majorant)
// are served from shared memory: 8 LDS + a software trilinear blend.  One 512-byte burst replaces eight dependent 4-byte
// gathers through the texture path, and a brick is fetched once per visit instead of once per look-up.
//
// Filtering: the reference samples with the texture unit's linear filter (clamp addressing; gpu_vdb.cpp:215-248).  The blend
// (vpt_texfilter.cuh) reproduces the unit's own rule, measured on the H100 (DESIGN.md section 3a): the coordinate truncated to 21
// fractional bits, integer corner weights that sum to 256 split z -> x -> y, the correctly rounded sum.  A pass rendered through the
// brick path flips no pixel against the texture path, so brick mode keeps per-seed parity with the reference kernel
// (tests/test_bricks_gpu.py); the texture path stays the default.
//
// Scope: the lean case of the direct integrator (one volume, no colour grid, no emission walk, no point lights); the host
// refuses fast mode for anything else.  Path start (start_path), control flow, random-number consumption and every other
// arithmetic step are the ones of k_trace (advance<true>, begin_ratio_walk, closest_object, hg_sample).
#pragma once

constexpr int kBrickThreads = 128;
constexpr int kBrickFloats = 128;                 // 125 texels + max + min + pad
constexpr int kBrickBytes = kBrickFloats * 4;

struct BrickArgs {
    const float* pool;                            // [nb.z][nb.y][nb.x][128]
    int nbx, nby, nbz;                            // bricks per axis
    int dimx, dimy, dimz;                         // voxels per axis
};

struct BrickSlot {
    uint32_t smem;                                // shared-memory address of my 512-byte slot
    uint32_t bar;                                 // shared-memory address of my mbarrier
    const float* data;                            // generic pointer to the slot
    int      resident;                            // linear brick id held by the slot (-1: none)
    uint32_t phase;                               // mbarrier phase parity to wait for next
};

VPT_DEV uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

VPT_DEV void brick_fetch(BrickSlot& bs, const float* src)
{
    // the slot was last READ through the generic proxy; order those reads before the async-proxy write that follows
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bs.bar), "r"(kBrickBytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(bs.smem), "l"(src), "r"(kBrickBytes), "r"(bs.bar) : "memory");
    uint32_t done = 0;
    while (!done) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(bs.bar), "r"(bs.phase) : "memory");
    }
    bs.phase ^= 1u;
}

// the software filter itself (coordinate rule, integer corner weights, blend): vpt_texfilter.cuh
using BrickCell = TexCell;
template <int kWeightMode>
VPT_DEV BrickCell brick_cell(float3 uvw, const BrickArgs& ba) { return tex_cell<kWeightMode>(uvw, ba.dimx, ba.dimy, ba.dimz); }

VPT_DEV int brick_id(const BrickCell& q, const BrickArgs& ba) { return ((q.k >> 2) * ba.nby + (q.j >> 2)) * ba.nbx + (q.i >> 2); }

// blend of the cell's eight texels inside a 5x5x5 brick at `brick`
template <int kWeightMode>
VPT_DEV float brick_blend(const float* brick, const BrickCell& q)
{
    const float* s = brick + ((q.k & 3) * 5 + (q.j & 3)) * 5 + (q.i & 3);
    return tex_blend<kWeightMode>(q, s[0], s[1], s[5], s[6], s[25], s[26], s[30], s[31]);
}

// the look-up at a normalised coordinate: stage the brick under it into the lane's slot unless it is the resident one, then blend
VPT_DEV float brick_sample(float3 uvw, const BrickArgs& ba, BrickSlot& bs, uint32_t& nfetch)
{
    const BrickCell q = brick_cell<kBrickWeightMode>(uvw, ba);
    const int id = brick_id(q, ba);
    if (id != bs.resident) {
        brick_fetch(bs, ba.pool + (size_t)id * kBrickFloats);
        bs.resident = id;
        nfetch++;
    }
    return brick_blend<kBrickWeightMode>(bs.data, q);
}

VPT_DEV float brick_density(const VolumeRec& v, float3 p, const BrickArgs& ba, BrickSlot& bs, uint32_t& nfetch)
{
    float3 uvw;
    if (!volume_coord(v, p, uvw)) return 0.0f;
    return brick_sample(uvw, ba, bs, nfetch);
}

// Diagnostic: software filter (three weight rules, bricks read straight from global memory) against the texture unit on `n`
// pseudo-random points of the unit cube.  out[mode * 4 + {0,1,2,3}] = max |d|, sum |d|, number of bit-identical results, n.
template <int kWeightMode>
VPT_DEV float brick_sample_global(float3 uvw, const BrickArgs& ba)
{
    const BrickCell q = brick_cell<kWeightMode>(uvw, ba);
    return brick_blend<kWeightMode>(ba.pool + (size_t)brick_id(q, ba) * kBrickFloats, q);
}

__global__ void k_sampler_compare(cudaTextureObject_t tex, const BrickArgs ba, int n, uint32_t seed, double* out)
{
    float mx[3] = { 0.f, 0.f, 0.f }; double sum[3] = { 0, 0, 0 }; unsigned long long same[3] = { 0, 0, 0 };
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const PhiloxBlock r = philox4x32_10((uint32_t)i, 0u, seed);
        const float3 uvw = f3(u32_to_unit(r.x), u32_to_unit(r.y), u32_to_unit(r.z));
        const float t = tex3D<float>(tex, uvw.x, uvw.y, uvw.z);
        const float s0 = brick_sample_global<0>(uvw, ba), s1 = brick_sample_global<1>(uvw, ba), s2 = brick_sample_global<2>(uvw, ba);
        const float d[3] = { fabsf(s0 - t), fabsf(s1 - t), fabsf(s2 - t) };
        const float sv[3] = { s0, s1, s2 };
        for (int m = 0; m < 3; ++m) { mx[m] = fmaxf(mx[m], d[m]); sum[m] += d[m]; same[m] += (__float_as_uint(sv[m]) == __float_as_uint(t)) ? 1ull : 0ull; }
    }
    for (int m = 0; m < 3; ++m) {
        for (int o = 16; o > 0; o >>= 1) {
            mx[m] = fmaxf(mx[m], __shfl_xor_sync(0xffffffffu, mx[m], o));
            sum[m] += __shfl_xor_sync(0xffffffffu, sum[m], o);
            same[m] += __shfl_xor_sync(0xffffffffu, same[m], o);
        }
        if ((threadIdx.x & 31) == 0) {
            // max of non-negative doubles == max of their bit patterns
            atomicMax(reinterpret_cast<unsigned long long*>(out + m * 4 + 0), (unsigned long long)__double_as_longlong((double)mx[m]));
            atomicAdd(out + m * 4 + 1, sum[m]);
            atomicAdd(out + m * 4 + 2, (double)same[m]);
        }
    }
}

// Diagnostic (vpt_debug_software_sample): the brick and cell samplers of the trace kernels at caller-chosen normalised points in [0, 1]^3.
// out2[2 p] = brick_sample (pool != 0), out2[2 p + 1] = cell_sample (cells != 0), 0 for the sampler not asked for.  Every thread owns a
// 512-byte slot and an mbarrier as in k_trace_brick and takes kSamplePointsPerLane CONSECUTIVE points, so a point list whose neighbours
// alternate between staying in a brick and leaving it runs both sides of the residency test.  64 slots = 32 KB of dynamic shared memory.
constexpr int kSampleThreads = 64;
constexpr int kSamplePointsPerLane = 32;

__global__ void __launch_bounds__(kSampleThreads)
k_software_sample(const BrickArgs ba, const float4* __restrict__ cells, const float* __restrict__ uvw, int n, float* __restrict__ out2)
{
    __shared__ __align__(8) unsigned long long bars[kSampleThreads];
    extern __shared__ __align__(128) float slots[];               // kSampleThreads x 128 floats
    BrickSlot bs;
    bs.data = slots + threadIdx.x * kBrickFloats; bs.smem = smem_addr(bs.data);
    bs.bar = smem_addr(&bars[threadIdx.x]); bs.resident = -1; bs.phase = 0u;
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(bs.bar) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();

    const int3 dims = make_int3(ba.dimx, ba.dimy, ba.dimz);
    const long long first = ((long long)blockIdx.x * kSampleThreads + threadIdx.x) * kSamplePointsPerLane;
    const long long last = min(first + kSamplePointsPerLane, (long long)n);
    uint32_t nfetch = 0;
    for (long long p = first; p < last; ++p) {
        const float3 q = f3(uvw[3 * p], uvw[3 * p + 1], uvw[3 * p + 2]);
        out2[2 * p] = ba.pool ? brick_sample(q, ba, bs, nfetch) : 0.0f;
        out2[2 * p + 1] = cells ? cell_sample(cells, dims, q) : 0.0f;
    }
}

// One tracking step, as walk_step<true> (vpt_trace.cuh) with the density fetched from the brick slot and the throughput kept in
// registers (one ray per lane here).
VPT_DEV void walk_step_brick(PathState& st, const FrameShared& fs, const FrameArgs& fa, const TraceConsts& tc, const SphereRec& sph,
                             const BrickArgs& ba, BrickSlot& bs, uint32_t& nlook, uint32_t& nfetch)
{
    const SceneTables& sc = fs.sc;
    const vpt_kernel_params& kp = fa.kp;
    int leaf = oct_locate_or_skip(fs.oct, sc, st.wpos, st.wdir);
    if (leaf == -2) leaf = oct_locate_or_skip(fs.oct, sc, st.wpos, st.wdir);
    if (leaf == -2) return;
    if (leaf == -1) { st.op = OP_GLUE; st.exit_reason = EX_OUTSIDE; return; }

    if (st.mode == W_DELTA) {
        float t_min, t_max, geo_dist = .0f;
        aabb_intersect(sc.root_pmin, sc.root_pmax, st.wpos, st.wdir, t_min, st.distance);
        if (!st.sphere_free && sphere_intersect(sph, st.wpos, st.wdir, geo_dist, t_max)) st.distance = geo_dist;
    }
    const float u = st.rng.next();
    const float l2 = __log2f(psub(1.0f, u));
    if (st.mode == W_DELTA) st.t = pfma(tc.inv_mult, pmul(tc.inv_max, pmul(l2, -0.693147182f)), st.t);
    else                    st.t = pfma(kp.tr_depth, pmul(tc.sigma_r_inv, pmul(l2, -0.693147182f)), st.t);
    if (st.t >= st.distance) { st.op = OP_GLUE; st.exit_reason = EX_DISTANCE; return; }

    st.wpos = madd3(st.wpos, st.wdir, st.t);
    if (!aabb_contains(sc.root_pmin, sc.root_pmax, st.wpos)) { st.op = OP_GLUE; st.exit_reason = EX_OUTSIDE; return; }

    nlook++;
    const float density = 0.0f + brick_density(fs.vol0, st.wpos, ba, bs, nfetch);
    if (st.mode == W_DELTA) {
        if (st.alpha < 1.0f) st.alpha += density;
        if (pmul(tc.inv_max, density) > st.rng.next()) {
            const vpt_kernel_params& kp = fa.kp;                    // throughput update as walk_step<true>; the state is in registers here
            const float3 Cd = fmax3(f3(0.0f), volume_color(fs.vol0, st.wpos));
            const int index = int(floorf(fminf(fmaxf((density * tc.inv_max * 255.0f / kp.emission_pivot), 0.0f), 255.0f)));
            const float3 density_color = reinterpret_cast<const float3*>(kp.density_color_texture)[index];
            st.beta *= (ld3(kp.albedo) * Cd * density_color / ld3(kp.extinction)) * float(kp.energy_inject);
            st.op = OP_GLUE; st.exit_reason = EX_SCATTER;
        }
    } else {
        st.trv = pmul(st.trv, pfma(-tc.sigma_r_inv, psub(density, tc.sigma_c), 1.0f));
        if (length(f3(st.trv)) < VPT_EPS) { st.op = OP_GLUE; st.exit_reason = EX_TR_DONE; }
    }
}

__global__ void __launch_bounds__(kBrickThreads, 3)
k_trace_brick(const FrameArgs fa, const BrickArgs ba)
{
    __shared__ FrameShared fs;
    __shared__ __align__(8) unsigned long long bars[kBrickThreads];
    extern __shared__ __align__(128) float slots[];               // kBrickThreads x 128 floats (opt-in dynamic shared memory)
    load_frame_shared(fs, fa.scene);
    const SceneTables& sc = fs.sc;
    const int lane = threadIdx.x & 31;
    const unsigned lt_mask = (1u << lane) - 1u;

    BrickSlot bs;
    bs.data = slots + threadIdx.x * kBrickFloats; bs.smem = smem_addr(bs.data);
    bs.bar = smem_addr(&bars[threadIdx.x]); bs.resident = -1; bs.phase = 0u;
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(bs.bar) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();

    const TraceConsts tc = make_trace_consts(sc, fa.kp);
    const SphereRec sph = load_sphere(fa.sphere);

    const unsigned q_count = *fa.queue_count;
    bool queue_dry = (q_count == 0);
    uint32_t nlook = 0, nfetch = 0, lane_steps = 0, warp_iters = 0, lane_ops = 0, warp_ops = 0, lane_rays = 0;
    PathState st;
    st.op = OP_IDLE;

    for (;;) {
        // ---- refill: one atomic per warp, one queue record per idle lane ------------------------------------------------
        const unsigned idle_lanes = __ballot_sync(0xffffffffu, st.op == OP_IDLE);
        if (!queue_dry && idle_lanes) {
            unsigned base = 0;
            const int leader = __ffs(idle_lanes) - 1;
            if (lane == leader) base = atomicAdd(fa.queue_head, (unsigned)__popc(idle_lanes));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (base + __popc(idle_lanes) >= q_count) queue_dry = true;
            const unsigned slot = base + __popc(idle_lanes & lt_mask);
            if (st.op == OP_IDLE && slot < q_count) {
                start_path<0>(st, fa, slot);
                ray_rng_init(st, fa, st.rng.k);
                lane_rays++;
            }
        }

        // ---- vote between the two code sites: the tracking step and the integrator's bookkeeping ---------------------------
        const int nS = __popc(__ballot_sync(0xffffffffu, st.op == OP_STEP));
        const int nV = __popc(__ballot_sync(0xffffffffu, st.op != OP_STEP && st.op != OP_IDLE));
        if ((nS | nV) == 0) {
            if (queue_dry) break;
            continue;
        }
        if (nV > 0 && (nV >= fa.sched_min_lanes || nS == 0 || nV > nS)) {
            if (st.op != OP_STEP && st.op != OP_IDLE) {
                if (st.op == OP_CLOSEST) {
                    st.obj_c = closest_object(sc, sph, st.pos, st.dir, st.tmin_c);
                    st.have_closest = true; st.op = OP_GLUE;
                }
                if (st.op == OP_GLUE) advance<true>(st, fs, fa, tc, sph);
                if (st.op == OP_TRBEGIN) begin_ratio_walk(st, fs, tc, sph);
                if (st.op == OP_FINISH) { write_sample<0, true>(st, fa); st.op = OP_IDLE; }
                lane_ops++;
            }
            warp_ops++;
            continue;
        }
        if (st.op == OP_STEP) { walk_step_brick(st, fs, fa, tc, sph, ba, bs, nlook, nfetch); lane_steps++; }
        warp_iters++;
    }

    if (fa.counters) {
        unsigned long long a = nlook, b = lane_steps, c = lane_ops, d = lane_rays, e = nfetch;
        for (int o = 16; o > 0; o >>= 1) {
            a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); c += __shfl_xor_sync(0xffffffffu, c, o);
            d += __shfl_xor_sync(0xffffffffu, d, o); e += __shfl_xor_sync(0xffffffffu, e, o);
        }
        if (lane == 0) {
            atomicAdd(fa.counters + 0, a); atomicAdd(fa.counters + 1, b); atomicAdd(fa.counters + 2, (unsigned long long)warp_iters);
            atomicAdd(fa.counters + 3, c); atomicAdd(fa.counters + 4, (unsigned long long)warp_ops); atomicAdd(fa.counters + 5, d);
            atomicAdd(fa.counters + 6, e);
        }
    }
}
