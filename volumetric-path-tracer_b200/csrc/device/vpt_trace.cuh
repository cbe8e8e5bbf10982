// vpt_trace.cuh -- k_trace: persistent wavefront over the hit queue, three rays per lane.
// (included from vpt_kernels.cu inside `namespace vpt`)
//
// Divergence is the enemy of this path: a ray needs a different heavy operation every few hundred
// instructions (closest-object test, tracking step, HG resampling, transmittance set-up, bookkeeping)
// and walks have geometric length.  One-ray-per-lane designs leave most lanes of a warp idle on each
// issued instruction.  Here every LANE owns kSlots = 3 rays, parked in shared memory (34 words each,
// word-major so that lane l only ever touches bank l, or in 16-byte groups: conflict-free, no inter-lane hand-over) and tagged,
// in registers, with the operation they wait for:
//
//     OP_STEP     one unified tracking step (delta / residual-ratio / emission walk)
//     OP_CLOSEST  nearest of {octree root box, sphere}            (reference get_closest_object)
//     OP_TRBEGIN  set-up of a residual-ratio transmittance walk   (reference Tr prologue)
//     OP_GLUE     integrator bookkeeping after a walk ended (HG resampling, NEE results, retirement)      OP_IDLE  free slot
//
// Each round the warp votes between two code sites: the STEPPING LOOP (a lane steps one of its walkers; when that walk
// ends it parks the ray and swaps in its next walker, so the step body keeps most lanes busy until the warp runs out of
// walkers) and a SERVICE ROUND (one parked ray per lane runs [closest-object test] -> the integrator's control flow
// `advance` -> [transmittance set-up], each block once in the code).  Free slots are refilled from the global ray queue
// with one atomic per warp.  The walk path moves 13 + 10 words of the record per swap and carries the packed flag word
// as is; the kernel is instantiated per integrator and in a "lean" form without multi-volume / emission / point-light
// code for the common scene (the kernel is fetch / issue bound: less code runs faster).
//
// Control flow restated from the reference direct integrator (render_kernel.cu:1760-1857) with three
// bit-exact shortcuts: (1) the depth pass replays the integrator's first walk on a copy of the RNG
// (:1859-1889), so it is taken from that walk instead of being run again; (2) the closest-object test
// at the end of a bounce and the one at the top of the next have identical inputs unless the sphere
// branch ran, so the result is reused (and the very first one comes from k_generate); (3) a bounce that
// finds nothing ahead makes every later bounce a no-op, so the path retires there.
#pragma once

enum WalkMode : int { W_DELTA = 1, W_RATIO = 2, W_EMIT = 3 };
enum Op : int { OP_IDLE = 0, OP_GLUE, OP_STEP, OP_CLOSEST, OP_TRBEGIN, OP_FINISH };
enum Phase : int {
    PH_BOUNCE_TOP = 0, PH_TOP_HAVE, PH_VOL_ITER, PH_AFTER_DELTA, PH_AFTER_HG, PH_VOL_DONE, PH_AFTER_TR,
    PH_POINT_NEXT, PH_EMISSION, PH_AFTER_EMIT, PH_AFTER_VOLUME, PH_AFTERVOL_HAVE, PH_SPHERE
};
enum ExitReason : int { EX_NONE = 0, EX_OUTSIDE, EX_DISTANCE, EX_SCATTER, EX_TR_DONE };
enum TrKind : int { TR_SUN = 0, TR_POINT = 1, TR_SPHERE = 2 };

// rays per lane: 3 (4 CTAs of 128 threads per SM, <= 128 registers) or 2: more warps in flight, the better trade when every look-up
// misses all caches; slower when the look-ups hit L2.  The generic kernels at 2 run 5 CTAs of 128 threads (<= 96 registers); the lean
// ones, whose stepping loop is bound by the latency of its look-ups, park a 29-word record and run the shape of VPT_LEAN2_SHAPE
// (trace_threads, trace_min_ctas, trace_smem_bytes in vpt_kernels.h; DESIGN.md section 4).

struct PathState {
    float3 pos, dir;      // the integrator's ray
    float3 org;           // camera-ray origin (depth reference, default env_pos); not stored: pinhole -> cam.origin, else queue_org[qslot]
    float3 beta, L;
    float  alpha;         // the reference's `tr` out-parameter (accumulated density, capped at 1 at the end)
    float  depth;
    float3 wpos, wdir;    // running walk (Tr and the emission walk run on copies of the ray)
    float  t, distance;
    float  trv, T_c;      // residual-ratio running value and control-variate factor
    float3 aux;           // emission accumulator | point-light accumulator | sphere normal (never live together)
    float  tmin_c;        // cached closest-object result
    int    obj_c;
    int    op, phase, mode, exit_reason, tr_kind;
    int    rd, vd, light_budget, light_index;
    bool   mi, first_walk, have_closest, sphere_bounced;
    bool   sphere_free;   // the running walk's line provably misses the sphere: its per-step intersection tests are skipped
    uint32_t lp, pass, qslot;
    uint32_t packed;      // word 30 as parked (walk path only: the stepping loop edits mode-independent bits in place)
    Rng    rng;
};

struct TraceConsts {
    float inv_max, inv_mult, sigma_c, sigma_r_inv;
    float3 sun_dir;
};

VPT_DEV TraceConsts make_trace_consts(const SceneTables& sc, const vpt_kernel_params& kp)
{
    TraceConsts tc;
    tc.inv_max = 1.0f / sc.max_extinction;
    tc.inv_mult = 1.0f / kp.density_mult;
    tc.sigma_c = sc.min_extinction;
    tc.sigma_r_inv = 1.0f / (sc.max_extinction - tc.sigma_c);
    tc.sun_dir = sun_direction(kp.azimuth, kp.elevation);
    return tc;
}

// The state of a path that has not started yet: throughput 1, no radiance, first bounce, first walk (camera ray in st.org / st.dir)
VPT_DEV void reset_path(PathState& st)
{
    st.pos = st.org;
    st.beta = f3(1.0f); st.L = f3(.0f); st.alpha = .0f; st.depth = .0f;
    st.wpos = st.pos; st.wdir = st.dir; st.aux = f3(0.f); st.t = 0.f; st.distance = 0.f; st.trv = 1.f; st.T_c = 1.f;
    st.mi = false; st.first_walk = true; st.sphere_bounced = false; st.rd = 1; st.vd = 1; st.light_budget = 0; st.light_index = 0;
    st.mode = W_DELTA; st.exit_reason = EX_NONE; st.tr_kind = TR_SUN; st.sphere_free = false;
}

// ---- light groups (the kGroups instantiations; DESIGN.md section 8d) -----------------------------------------------------------
// Every `L +=` site of those instantiations also adds its term to the ray's sum of that light class, kept in the sample scratch at the
// ray's own sample slot: one ray per slot, so a plain read-modify-write (no atomics, deterministic).  ptxas contracts a single-use product
// into the following add, and a product used for L AND for the group is no longer single-use, so both updates are pinned to the fma the
// instantiation without groups compiles to: L + a * b -> fma(a, b, L).
VPT_DEV const LightGroups* lg_of(const LightGroups& a) { return &a; }
VPT_DEV const LightGroups* lg_of(const LightGroups& a, const MatteIds&) { return &a; }
VPT_DEV float3 pfma3(const float3 a, const float3 b, const float3 c) { return f3(pfma(a.x, b.x, c.x), pfma(a.y, b.y, c.y), pfma(a.z, b.z, c.z)); }
VPT_DEV size_t group_slot(const PathState& st, const FrameArgs& fa) { return (size_t)st.pass * fa.geom.n_local + ray_local_pixel(fa.geom, st.lp); }
VPT_DEV void group_fma(const LightGroups* lg, const size_t s, const int group, const float3 a, const float3 b) {
    float* p = lg->planes + (size_t)(group * 3) * lg->stride + s;
    const size_t n = lg->stride;
    p[0] = pfma(a.x, b.x, p[0]); p[n] = pfma(a.y, b.y, p[n]); p[2 * n] = pfma(a.z, b.z, p[2 * n]);
}
VPT_DEV void group_add(const LightGroups* lg, const size_t s, const int group, const float3 a) {
    float* p = lg->planes + (size_t)(group * 3) * lg->stride + s;
    const size_t n = lg->stride;
    p[0] = padd(p[0], a.x); p[n] = padd(p[n], a.y); p[2 * n] = padd(p[2 * n], a.z);
}

// ---- instance mattes (the instantiations whose pack ends with a MatteIds; DESIGN.md section 8l) ------------------------------------
// The id of the camera ray's first collision goes to the id plane at the ray's sample slot.  The walks, their draws and walk_step itself
// are those of the instantiations without mattes (a template parameter more on walk_step moved a stack store of the group and volumetric
// kernels): the instance comes from the acceptance draw u the walk already made, regenerated from the counter-based stream.
VPT_DEV const MatteIds* mt_of(const MatteIds& m) { return &m; }
VPT_DEV const MatteIds* mt_of(const LightGroups&, const MatteIds& m) { return &m; }
VPT_DEV const MatteIds* matte_ids(const MatteIds* m) { return m; }
// the last draw of the stream: at PH_AFTER_DELTA / VP_AFTER_DELTA after an accepted collision, the u of the accepting test (walk_step ends
// the walk there, and nothing draws before the id is taken).  Philox is counter-based: the copy re-evaluates draw k - 1, and `rng` is untouched.
VPT_DEV float last_draw(const Rng& rng) { Rng r = rng; r.k -= 1u; return r.next(); }
// the instance of an accepted collision at p in `leaf` with acceptance draw u: the first entry i of the leaf's list whose density prefix
// (the float sum over entries 0..i in list order, as leaf_density adds them) passes the walk's test pmul(inv_max, prefix) > u.  The last
// prefix is the density the walk accepted, bit for bit, so some entry always passes (negative densities included).
VPT_DEV uint32_t collision_instance(const SceneTables& sc, const int leaf, const float3 p, const float u, const float inv_max)
{
    if (sc.single_volume) return 0u;
    const LeafList lst = leaf_list_of(sc, leaf);
    float prefix = 0.0f;
    for (uint32_t i = 0; i < lst.n; ++i) {
        prefix += volume_density(sc.volumes[lst.idx[i]], p);
        if (pmul(inv_max, prefix) > u) return (uint32_t)lst.idx[i];
    }
    return lst.n ? (uint32_t)lst.idx[lst.n - 1] : 0u;           // not reached after an accepted collision
}

// ---- ray record <-> registers ------------------------------------------------------------------------------
// pool layout: word w of slot j of lane l at pool[w * kPool + j * 32 + l]  (bank == lane: conflict-free)
template <int kPool>                                             // rays per warp = 32 * rays per lane
struct PoolView {
    float* w;                                                    // this warp's kRayWords * kPool words, already offset by the lane
    VPT_DEV float& f(int word, int slot) const { return w[word * kPool + slot * 32]; }
    VPT_DEV uint32_t& u(int word, int slot) const { return reinterpret_cast<uint32_t*>(w)[word * kPool + slot * 32]; }
};

template <class PV>
VPT_DEV void store_ray(const PV& pv, int s, const PathState& st)
{
    pv.f(0, s) = st.pos.x;  pv.f(1, s) = st.pos.y;  pv.f(2, s) = st.pos.z;
    pv.f(3, s) = st.dir.x;  pv.f(4, s) = st.dir.y;  pv.f(5, s) = st.dir.z;
    pv.f(6, s) = st.L.x;    pv.f(7, s) = st.L.y;    pv.f(8, s) = st.L.z;
    pv.f(9, s) = st.beta.x; pv.f(10, s) = st.beta.y; pv.f(11, s) = st.beta.z;
    pv.f(12, s) = st.wpos.x; pv.f(13, s) = st.wpos.y; pv.f(14, s) = st.wpos.z;
    pv.f(15, s) = st.wdir.x; pv.f(16, s) = st.wdir.y; pv.f(17, s) = st.wdir.z;
    pv.f(18, s) = st.aux.x; pv.f(19, s) = st.aux.y; pv.f(20, s) = st.aux.z;
    pv.f(21, s) = st.alpha; pv.f(22, s) = st.depth; pv.f(23, s) = st.t; pv.f(24, s) = st.distance;
    pv.f(25, s) = st.trv;   pv.f(26, s) = st.T_c;   pv.f(27, s) = st.tmin_c;
    pv.u(28, s) = st.rng.k; pv.u(29, s) = st.lp;
    pv.u(30, s) = (uint32_t)st.phase | ((uint32_t)st.mode << 4) | ((uint32_t)st.exit_reason << 6) | ((uint32_t)st.tr_kind << 9) |
                  ((uint32_t)st.obj_c << 11) | ((uint32_t)st.mi << 13) | ((uint32_t)st.first_walk << 14) | ((uint32_t)st.have_closest << 15) |
                  ((uint32_t)st.sphere_bounced << 16) | ((uint32_t)st.sphere_free << 17) | (st.pass << 18);
    pv.u(31, s) = (uint32_t)(st.rd & 0xffff) | ((uint32_t)(st.vd & 0xffff) << 16);
    pv.u(32, s) = (uint32_t)(st.light_budget & 0xff) | ((uint32_t)st.light_index << 8);
    pv.u(33, s) = st.qslot;
}

// the camera-ray origin of queue record `slot`: its own under a thin lens, the camera's for a pinhole
VPT_DEV float3 ray_origin(const FrameArgs& fa, uint32_t slot)
{
    return fa.thin_lens ? f3(__ldg(fa.queue_aux + slot).x, __ldg(fa.queue_aux + slot).y, __ldg(fa.queue_aux + slot).z) : ld3(fa.cam.origin);
}

VPT_DEV void ray_rng_init(PathState& st, const FrameArgs& fa, uint32_t k)
{
    uint32_t idx = st.lp;                                    // the ray's pixel word (vpt_frame.cuh): the pixel index itself for one rank
    if (fa.geom.n_ranks > 1) idx = ray_global_pixel(fa.geom, st.lp);
    st.rng.init(idx, fa.kp.iteration + st.pass, k);
}

template <class PV>
VPT_DEV void load_ray(const PV& pv, int s, PathState& st, const FrameArgs& fa)
{
    st.pos = f3(pv.f(0, s), pv.f(1, s), pv.f(2, s));    st.dir = f3(pv.f(3, s), pv.f(4, s), pv.f(5, s));
    st.L = f3(pv.f(6, s), pv.f(7, s), pv.f(8, s));      st.beta = f3(pv.f(9, s), pv.f(10, s), pv.f(11, s));
    st.wpos = f3(pv.f(12, s), pv.f(13, s), pv.f(14, s)); st.wdir = f3(pv.f(15, s), pv.f(16, s), pv.f(17, s));
    st.aux = f3(pv.f(18, s), pv.f(19, s), pv.f(20, s));
    st.alpha = pv.f(21, s); st.depth = pv.f(22, s); st.t = pv.f(23, s); st.distance = pv.f(24, s);
    st.trv = pv.f(25, s);   st.T_c = pv.f(26, s);   st.tmin_c = pv.f(27, s);
    const uint32_t k = pv.u(28, s); st.lp = pv.u(29, s);
    const uint32_t a = pv.u(30, s), b = pv.u(31, s), c = pv.u(32, s);
    st.phase = a & 15; st.mode = (a >> 4) & 3; st.exit_reason = (a >> 6) & 7; st.tr_kind = (a >> 9) & 3; st.obj_c = (a >> 11) & 3;
    st.mi = (a >> 13) & 1; st.first_walk = (a >> 14) & 1; st.have_closest = (a >> 15) & 1; st.sphere_bounced = (a >> 16) & 1; st.sphere_free = (a >> 17) & 1; st.pass = a >> 18;
    st.rd = b & 0xffff; st.vd = b >> 16;
    st.light_budget = (int)(int8_t)(c & 0xff); st.light_index = c >> 8;
    st.qslot = pv.u(33, s);
    st.org = ray_origin(fa, st.qslot);
    ray_rng_init(st, fa, k);
}

// A walk only touches part of the record (13 words in, 10 out instead of 34 each way) and only two of the eleven fields packed
// in word 30: the packed word is carried as is and patched on the way out (unpacking/packing everything cost 5 % of the kernel's
// instructions).  beta is not carried either: the one event that changes it (a scatter) updates it in place in shared memory.
constexpr uint32_t kExitMask = 7u << 6;
template <class PV>
VPT_DEV void load_walk(const PV& pv, int s, PathState& st, const FrameArgs& fa)
{
    st.wpos = f3(pv.f(12, s), pv.f(13, s), pv.f(14, s)); st.wdir = f3(pv.f(15, s), pv.f(16, s), pv.f(17, s));
    st.aux = f3(pv.f(18, s), pv.f(19, s), pv.f(20, s));
    st.alpha = pv.f(21, s); st.t = pv.f(23, s); st.distance = pv.f(24, s); st.trv = pv.f(25, s);
    const uint32_t k = pv.u(28, s); st.lp = pv.u(29, s);
    const uint32_t a = pv.u(30, s);
    st.packed = a;
    st.mode = (a >> 4) & 3; st.exit_reason = (a >> 6) & 7; st.sphere_free = (a >> 17) & 1; st.pass = a >> 18;
    ray_rng_init(st, fa, k);
}

template <class PV>
VPT_DEV void store_walk(const PV& pv, int s, const PathState& st)
{
    pv.f(12, s) = st.wpos.x; pv.f(13, s) = st.wpos.y; pv.f(14, s) = st.wpos.z;
    pv.f(18, s) = st.aux.x; pv.f(19, s) = st.aux.y; pv.f(20, s) = st.aux.z;
    pv.f(21, s) = st.alpha; pv.f(23, s) = st.t; pv.f(25, s) = st.trv;
    pv.u(28, s) = st.rng.k;
    pv.u(30, s) = (st.packed & ~kExitMask) | ((uint32_t)st.exit_reason << 6);
}

// The headline kernels (lean, 3 rays per lane) park the same 34 words in eight 16-byte groups and one 8-byte group, each moved by one
// 128-bit / 64-bit shared-memory access (a service round moves 9 groups each way instead of 34 words, a walk swap 4 + 3 groups instead of 16 + 11 words):
//   G_WPOS {wpos, t}   G_WDIR {wdir, distance}   G_AUX {aux, alpha}   G_WALK {trv, rng.k, lp, packed word}      (the walk's groups)
//   G_POS {pos, depth}   G_DIR {dir, T_c}   G_L {L, tmin_c}   G_BETA {beta, qslot}   and the 8-byte {rd | vd, light word}
// Group g of slot j of lane l at vector index (g * kSlots + j) * 32 + l of the warp's pool: a quarter-warp's 128-bit access covers 128
// contiguous bytes (conflict-free).  The other kernels keep the word-major view above: with 128-bit moves the generic kernel ran slower on
// the fireball (config 3) and the kernels at 2 rays per lane spilled more.
enum RayGroup : int { G_WPOS = 0, G_WDIR, G_AUX, G_WALK, G_POS, G_DIR, G_L, G_BETA, kRayGroups4 };
static_assert(kRayGroups4 * 4 + 2 == kRayWords, "eight 16-byte groups and one 8-byte group per ray");
template <int kSlots>
struct PoolGroups {
    float4* q;                                                   // this warp's 16-byte groups, already offset by the lane
    float2* h;                                                   // its 8-byte groups, already offset by the lane
    VPT_DEV float4& g(int group, int slot) const { return q[(group * kSlots + slot) * 32]; }
    VPT_DEV float2& g2(int slot) const { return h[slot * 32]; }
};
VPT_DEV float4 f4(const float3 v, const float w) { return make_float4(v.x, v.y, v.z, w); }
VPT_DEV float3 xyz(const float4 v) { return f3(v.x, v.y, v.z); }

template <int kSlots>
VPT_DEV void store_ray(const PoolGroups<kSlots>& pv, int s, const PathState& st)
{
    const uint32_t a = (uint32_t)st.phase | ((uint32_t)st.mode << 4) | ((uint32_t)st.exit_reason << 6) | ((uint32_t)st.tr_kind << 9) |
                       ((uint32_t)st.obj_c << 11) | ((uint32_t)st.mi << 13) | ((uint32_t)st.first_walk << 14) | ((uint32_t)st.have_closest << 15) |
                       ((uint32_t)st.sphere_bounced << 16) | ((uint32_t)st.sphere_free << 17) | (st.pass << 18);
    pv.g(G_WPOS, s) = f4(st.wpos, st.t);
    pv.g(G_WDIR, s) = f4(st.wdir, st.distance);
    pv.g(G_AUX, s) = f4(st.aux, st.alpha);
    pv.g(G_WALK, s) = make_float4(st.trv, __uint_as_float(st.rng.k), __uint_as_float(st.lp), __uint_as_float(a));
    pv.g(G_POS, s) = f4(st.pos, st.depth);
    pv.g(G_DIR, s) = f4(st.dir, st.T_c);
    pv.g(G_L, s) = f4(st.L, st.tmin_c);
    pv.g(G_BETA, s) = f4(st.beta, __uint_as_float(st.qslot));
    pv.g2(s) = make_float2(__uint_as_float((uint32_t)(st.rd & 0xffff) | ((uint32_t)(st.vd & 0xffff) << 16)),
                           __uint_as_float((uint32_t)(st.light_budget & 0xff) | ((uint32_t)st.light_index << 8)));
}

template <int kSlots>
VPT_DEV void load_ray(const PoolGroups<kSlots>& pv, int s, PathState& st, const FrameArgs& fa)
{
    const float4 gwp = pv.g(G_WPOS, s), gwd = pv.g(G_WDIR, s), gax = pv.g(G_AUX, s), gwk = pv.g(G_WALK, s);
    const float4 gp = pv.g(G_POS, s), gd = pv.g(G_DIR, s), gl = pv.g(G_L, s), gb = pv.g(G_BETA, s);
    const float2 gc = pv.g2(s);
    st.pos = xyz(gp);    st.depth = gp.w;    st.dir = xyz(gd);   st.T_c = gd.w;
    st.L = xyz(gl);      st.tmin_c = gl.w;   st.beta = xyz(gb);  st.qslot = __float_as_uint(gb.w);
    st.wpos = xyz(gwp);  st.t = gwp.w;       st.wdir = xyz(gwd); st.distance = gwd.w;
    st.aux = xyz(gax);   st.alpha = gax.w;
    st.trv = gwk.x;
    const uint32_t k = __float_as_uint(gwk.y); st.lp = __float_as_uint(gwk.z);
    const uint32_t a = __float_as_uint(gwk.w), b = __float_as_uint(gc.x), c = __float_as_uint(gc.y);
    st.phase = a & 15; st.mode = (a >> 4) & 3; st.exit_reason = (a >> 6) & 7; st.tr_kind = (a >> 9) & 3; st.obj_c = (a >> 11) & 3;
    st.mi = (a >> 13) & 1; st.first_walk = (a >> 14) & 1; st.have_closest = (a >> 15) & 1; st.sphere_bounced = (a >> 16) & 1; st.sphere_free = (a >> 17) & 1; st.pass = a >> 18;
    st.rd = b & 0xffff; st.vd = b >> 16;
    st.light_budget = (int)(int8_t)(c & 0xff); st.light_index = c >> 8;
    st.org = ray_origin(fa, st.qslot);
    ray_rng_init(st, fa, k);
}

template <int kSlots>
VPT_DEV void load_walk(const PoolGroups<kSlots>& pv, int s, PathState& st, const FrameArgs& fa)
{
    const float4 gwp = pv.g(G_WPOS, s), gwd = pv.g(G_WDIR, s), gax = pv.g(G_AUX, s), gwk = pv.g(G_WALK, s);
    st.wpos = xyz(gwp); st.t = gwp.w; st.wdir = xyz(gwd); st.distance = gwd.w;
    st.aux = xyz(gax);  st.alpha = gax.w;
    st.trv = gwk.x;
    const uint32_t k = __float_as_uint(gwk.y); st.lp = __float_as_uint(gwk.z);
    const uint32_t a = __float_as_uint(gwk.w);
    st.packed = a;
    st.mode = (a >> 4) & 3; st.exit_reason = (a >> 6) & 7; st.sphere_free = (a >> 17) & 1; st.pass = a >> 18;
    ray_rng_init(st, fa, k);
}

template <int kSlots>
VPT_DEV void store_walk(const PoolGroups<kSlots>& pv, int s, const PathState& st)
{
    pv.g(G_WPOS, s) = f4(st.wpos, st.t);
    pv.g(G_AUX, s) = f4(st.aux, st.alpha);
    pv.g(G_WALK, s) = make_float4(st.trv, __uint_as_float(st.rng.k), __uint_as_float(st.lp),
                                  __uint_as_float((st.packed & ~kExitMask) | ((uint32_t)st.exit_reason << 6)));
}

// The lean kernels at 2 rays per lane park 29 words, word-major as PoolView (DESIGN.md section 4): six words of the 34 hold nothing a
// lean path needs across a park, so they are not stored, and one word is added (word 28, below).  The frame stays bit for bit what the
// 34-word record gives:
//   wdir     a lean walk is either the delta walk along the path's dir (PH_VOL_ITER, start_path) or a transmittance walk along
//            tc.sun_dir (PH_VOL_DONE, PH_SPHERE; begin_ratio_walk reads wdir and never writes it): load_walk takes it from `mode`.  A
//            service round needs none (advance assigns wdir before each walk, and begin_ratio_walk runs in the round that asked for it).
//   light    no point lights: light_budget and light_index stay 0.
//   T_c      live from begin_ratio_walk to PH_AFTER_TR only, where it is 1 or expf(-sigma_c * distance) of the walk's unchanged distance:
//            bit 24 of the packed word says which, and load_ray recomputes it (the same expression on the same inputs).
//   tmin_c   read only in the service round of the closest-object test that computed it, or in a fresh path's first round (parked at
//            PH_BOUNCE_TOP with k_generate's test); trv is dead there (begin_ratio_walk sets it before any read), so the two share word 22.
// pass < 64 (start_path) leaves bits 24..31 of the packed word free; rd and vd keep their 16 bits each.
//   0-2 pos   3-5 dir   6-8 L   9-11 beta   12-14 wpos   15-17 aux   18 alpha   19 depth   20 t   21 distance   22 trv | tmin_c
//   23 rng.k   24 lp   25 packed word   26 rd | vd   27 qslot   28 rng.key
// Word 28, the ray's Philox key (its global pixel), is the one word more than the 34-word record needs: a walk swap keys the stream from
// it instead of from the pixel word, so the stepping loop holds no multi-rank row arithmetic (which spilled at 72 registers).
template <int kPool>
struct PoolLean {
    float* w;                                                    // this warp's kLeanRayWords * kPool words, already offset by the lane
    float3 sun_dir;                                              // TraceConsts: a transmittance walk's direction
    float sigma_c;                                               // ... and the control variate's extinction of T_c
    VPT_DEV float& f(int word, int slot) const { return w[word * kPool + slot * 32]; }
    VPT_DEV uint32_t& u(int word, int slot) const { return reinterpret_cast<uint32_t*>(w)[word * kPool + slot * 32]; }
};
constexpr uint32_t kTcBit = 1u << 24;                            // packed word of PoolLean: T_c is expf(-sigma_c * distance), not 1

template <int kPool>
VPT_DEV void store_ray(const PoolLean<kPool>& pv, int s, const PathState& st)
{
    pv.f(0, s) = st.pos.x;  pv.f(1, s) = st.pos.y;  pv.f(2, s) = st.pos.z;
    pv.f(3, s) = st.dir.x;  pv.f(4, s) = st.dir.y;  pv.f(5, s) = st.dir.z;
    pv.f(6, s) = st.L.x;    pv.f(7, s) = st.L.y;    pv.f(8, s) = st.L.z;
    pv.f(9, s) = st.beta.x; pv.f(10, s) = st.beta.y; pv.f(11, s) = st.beta.z;
    pv.f(12, s) = st.wpos.x; pv.f(13, s) = st.wpos.y; pv.f(14, s) = st.wpos.z;
    pv.f(15, s) = st.aux.x; pv.f(16, s) = st.aux.y; pv.f(17, s) = st.aux.z;
    pv.f(18, s) = st.alpha; pv.f(19, s) = st.depth; pv.f(20, s) = st.t; pv.f(21, s) = st.distance;
    pv.f(22, s) = st.phase == PH_BOUNCE_TOP ? st.tmin_c : st.trv;
    pv.u(23, s) = st.rng.k; pv.u(24, s) = st.lp;
    pv.u(25, s) = (uint32_t)st.phase | ((uint32_t)st.mode << 4) | ((uint32_t)st.exit_reason << 6) | ((uint32_t)st.tr_kind << 9) |
                  ((uint32_t)st.obj_c << 11) | ((uint32_t)st.mi << 13) | ((uint32_t)st.first_walk << 14) | ((uint32_t)st.have_closest << 15) |
                  ((uint32_t)st.sphere_bounced << 16) | ((uint32_t)st.sphere_free << 17) | (st.pass << 18) | (st.T_c != 1.0f ? kTcBit : 0u);
    pv.u(26, s) = (uint32_t)(st.rd & 0xffff) | ((uint32_t)(st.vd & 0xffff) << 16);
    pv.u(27, s) = st.qslot; pv.u(28, s) = st.rng.key;
}

template <int kPool>
VPT_DEV void load_ray(const PoolLean<kPool>& pv, int s, PathState& st, const FrameArgs& fa)
{
    st.pos = f3(pv.f(0, s), pv.f(1, s), pv.f(2, s));    st.dir = f3(pv.f(3, s), pv.f(4, s), pv.f(5, s));
    st.L = f3(pv.f(6, s), pv.f(7, s), pv.f(8, s));      st.beta = f3(pv.f(9, s), pv.f(10, s), pv.f(11, s));
    st.wpos = f3(pv.f(12, s), pv.f(13, s), pv.f(14, s)); st.aux = f3(pv.f(15, s), pv.f(16, s), pv.f(17, s));
    st.alpha = pv.f(18, s); st.depth = pv.f(19, s); st.t = pv.f(20, s); st.distance = pv.f(21, s);
    st.trv = pv.f(22, s); st.tmin_c = st.trv;
    const uint32_t k = pv.u(23, s); st.lp = pv.u(24, s);
    const uint32_t a = pv.u(25, s), b = pv.u(26, s);
    st.phase = a & 15; st.mode = (a >> 4) & 3; st.exit_reason = (a >> 6) & 7; st.tr_kind = (a >> 9) & 3; st.obj_c = (a >> 11) & 3;
    st.mi = (a >> 13) & 1; st.first_walk = (a >> 14) & 1; st.have_closest = (a >> 15) & 1; st.sphere_bounced = (a >> 16) & 1; st.sphere_free = (a >> 17) & 1;
    st.pass = (a >> 18) & 63u;
    st.T_c = (a & kTcBit) ? expf(-pv.sigma_c * st.distance) : 1.0f;   // begin_ratio_walk's expression
    st.rd = b & 0xffff; st.vd = b >> 16;
    st.light_budget = 0; st.light_index = 0;
    st.qslot = pv.u(27, s);
    st.org = ray_origin(fa, st.qslot);
    st.rng.init(pv.u(28, s), fa.kp.iteration + st.pass, k);
}

// a walk loads 13 words (wpos, dir unless it is a transmittance walk, alpha, t, distance, trv, rng.k, rng.key, packed) and stores 8: the lean
// walk changes no aux, and its T_c bit rides in the packed word
template <int kPool>
VPT_DEV void load_walk(const PoolLean<kPool>& pv, int s, PathState& st, const FrameArgs& fa)
{
    const uint32_t a = pv.u(25, s);
    st.packed = a;
    st.mode = (a >> 4) & 3; st.exit_reason = (a >> 6) & 7; st.sphere_free = (a >> 17) & 1; st.pass = (a >> 18) & 63u;
    st.wpos = f3(pv.f(12, s), pv.f(13, s), pv.f(14, s));
    st.wdir = st.mode == W_DELTA ? f3(pv.f(3, s), pv.f(4, s), pv.f(5, s)) : pv.sun_dir;
    st.alpha = pv.f(18, s); st.t = pv.f(20, s); st.distance = pv.f(21, s); st.trv = pv.f(22, s);
    st.rng.init(pv.u(28, s), fa.kp.iteration + st.pass, pv.u(23, s));   // (a walk reads no pixel word)
}

template <int kPool>
VPT_DEV void store_walk(const PoolLean<kPool>& pv, int s, const PathState& st)
{
    pv.f(12, s) = st.wpos.x; pv.f(13, s) = st.wpos.y; pv.f(14, s) = st.wpos.z;
    pv.f(18, s) = st.alpha; pv.f(20, s) = st.t; pv.f(22, s) = st.trv;
    pv.u(23, s) = st.rng.k;
    pv.u(25, s) = (st.packed & ~kExitMask) | ((uint32_t)st.exit_reason << 6);
}

// Density of volume 0 from its cell table (vpt_cells_create): the eight corner texels of the cell under the point are 32 contiguous,
// aligned bytes -- one DRAM sector per look-up instead of the four or five a 2x2x2 footprint costs in the tiled texture array --
// blended with the texture unit's own arithmetic (vpt_texfilter.cuh).  On the 1024^3 grid DRAM traffic falls to the algorithmic 32 B per
// look-up (DESIGN.md 3a): an experiment kept as an instrument, not a faster path.  cell_sample: the look-up at a normalised coordinate in a
// table of dims texels (also vpt_debug_software_sample's); cell_density: at a world point.
VPT_DEV float cell_sample(const float4* table, int3 dims, float3 uvw)
{
    const TexCell q = tex_cell<0>(uvw, dims.x, dims.y, dims.z);
    const float4* c = table + 2 * (((size_t)q.k * (size_t)dims.y + (size_t)q.j) * (size_t)dims.x + (size_t)q.i);
    const float4 lo = __ldg(c), hi = __ldg(c + 1);
    return tex_blend<0>(q, lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w);
}

VPT_DEV float cell_density(const FrameArgs& fa, const VolumeRec& v, float3 p)
{
    float3 uvw;
    if (!volume_coord(v, p, uvw)) return .0f;
    return cell_sample(fa.cell_table, make_int3(fa.cell_nx, fa.cell_ny, fa.cell_nz), uvw);
}

// ---- OP_STEP -------------------------------------------------------------------------------------------------
// kLean: single volume, no emission walk, no point lights -- the headline configuration; those features' code is compiled out
// of that instantiation (smaller hot loop: the kernel is fetch-stall bound)
// the per-step sphere test of a delta walk is rare (only lines that may hit the sphere): out of line, it keeps the hot loop shorter
__device__ __noinline__ bool sphere_intersect_cold(const SphereRec& s, float3 ray_pos, float3 ray_dir, float& t_min, float& t_max) { return sphere_intersect(s, ray_pos, ray_dir, t_min, t_max); }
// hop statistics of k_trace (counters [8..11]): hops of delta / ratio / emission walks, walks ended by "empty ahead"
struct HopStats { uint32_t delta, ratio, emit, ahead; };

// kAhead (the lean k_trace only; the generic instantiations and the level (A) entry keep it off, DESIGN.md section 8j): end walks at an
// empty node from which no populated leaf lies ahead (`ea`).
//   Ratio walks: hops draw nothing and change nothing but wpos, so the walk would end outside the box with the same trv and Philox
//   position; finish_ratio_walk never reads wpos.
//   Delta walks whose line provably misses the sphere: such a walk leaves the box with no scatter and no draw, and the path then retires
//   whatever volume_depth and ray_depth are (quirk Q21, PH_AFTER_DELTA .. PH_AFTER_VOLUME) with its L, beta, dir, depth (0 when the first
//   walk ends so) and the first walk's doubled alpha; its position is never written.  So the walk finishes the path here: the first-walk
//   alpha update, then OP_FINISH.
template <bool kLean, bool kCells = false, bool kAhead = false>
VPT_DEV void walk_step(PathState& st, const FrameShared& fs, const FrameArgs& fa, const TraceConsts& tc, const SphereRec& sph, uint32_t& nlook,
                       float* beta = nullptr, int beta_stride = 0,   // kLean: the path's throughput in the parked record (x, y, z one stride
                                                                     // apart; stride 1: a 16-byte group of PoolGroups)
                       const EmptyAhead* ea = nullptr, HopStats* hs = nullptr)
{
    const SceneTables& sc = fs.sc;
    const vpt_kernel_params& kp = fa.kp;
    // ONE point location per call: an empty node is hopped over (no draw consumed) and the call returns.  A second and a third in-line copy
    // were slower -- the kernel is bound by instruction fetch, every copy of the octree descent in the hot loop costs more than the
    // iterations it saves.
    int leaf = oct_locate_or_skip<false, kAhead>(fs.oct, sc, st.wpos, st.wdir, ea, st.mode != W_DELTA || st.sphere_free);
#if defined(VPT_WALK_HOPS) && VPT_WALK_HOPS >= 2
    if (leaf == -2) leaf = oct_locate_or_skip(fs.oct, sc, st.wpos, st.wdir);
#endif
    if (leaf == -2) {
        if (kAhead) { hs->delta += st.mode == W_DELTA; hs->ratio += st.mode == W_RATIO; }   // (a lean kernel runs no emission walk)
        return;
    }
    if (leaf == -1) { st.op = OP_GLUE; st.exit_reason = EX_OUTSIDE; return; }
    if (kAhead && leaf == -3) {
        hs->ahead++;
        st.op = OP_GLUE; st.exit_reason = EX_OUTSIDE;
        if (st.mode == W_DELTA) {
            if (((st.packed >> 14) & 1u) && st.alpha < 1.0f) st.alpha += st.alpha;   // first walk: the depth pass's replay (depth stays 0)
            st.op = OP_FINISH;
        }
        return;
    }

    if (st.mode == W_DELTA) {
        // distance to the box exit (or to the sphere) from the CURRENT position, every step (:1647-1651)
        float t_min, t_max, geo_dist = .0f;
        aabb_intersect(sc.root_pmin, sc.root_pmax, st.wpos, st.wdir, t_min, st.distance);
        if (!st.sphere_free && sphere_intersect_cold(sph, st.wpos, st.wdir, geo_dist, t_max)) st.distance = geo_dist;
    }
    const float u = st.rng.next();
    // t -= log(1-u) * a * b, as the reference build evaluates it: fma(b, a * (lg2(1-u) * -ln2), t)
    const float l2 = __log2f(psub(1.0f, u));
    if (st.mode == W_DELTA)      st.t = pfma(tc.inv_mult, pmul(tc.inv_max, pmul(l2, -0.693147182f)), st.t);
    else if (kLean || st.mode == W_RATIO) st.t = pfma(kp.tr_depth, pmul(tc.sigma_r_inv, pmul(l2, -0.693147182f)), st.t);
    else st.t = pfma(-pmul(pmul(pmul(l2, 0.693147182f), tc.inv_max), kp.tr_depth), 1.0f / kp.extinction.x, st.t);   // fma(-(log*a*b), rcp(ext), t): reference SASS
    if ((kLean || st.mode != W_EMIT) && st.t >= st.distance) { st.op = OP_GLUE; st.exit_reason = EX_DISTANCE; return; }

    st.wpos = madd3(st.wpos, st.wdir, st.t);                  // cumulative t, never reset (quirk Q2)
    if (!aabb_contains(sc.root_pmin, sc.root_pmax, st.wpos)) { st.op = OP_GLUE; st.exit_reason = EX_OUTSIDE; return; }

    nlook++;
    if (!kLean && st.mode == W_EMIT) {
        st.aux += leaf_emission(sc, fs.vol0, leaf, st.wpos, reinterpret_cast<const float3*>(kp.emission_texture), kp.emission_pivot, kp.emission_scale);
        return;
    }
    const float density = kLean ? 0.0f + (kCells ? cell_density(fa, fs.vol0, st.wpos) : volume_density(fs.vol0, st.wpos)) : leaf_density(sc, fs.vol0, leaf, st.wpos);
    if (st.mode == W_DELTA) {
        if (st.alpha < 1.0f) st.alpha += density;
        if (pmul(tc.inv_max, density) > st.rng.next()) {
            if (kLean) {
                // single volume: the colour terms are two cached loads; updating the parked throughput here was faster than a
                // deferred update on the headline frame
                const float3 Cd = fmax3(f3(0.0f), volume_color(fs.vol0, st.wpos));
                const int index = int(floorf(fminf(fmaxf((density * tc.inv_max * 255.0f / kp.emission_pivot), 0.0f), 255.0f)));
                const float3 density_color = reinterpret_cast<const float3*>(kp.density_color_texture)[index];
                if (beta_stride == 1) {                             // one 128-bit read-modify-write of the group (qslot rides along)
                    float4* g = reinterpret_cast<float4*>(beta);
                    const float4 gb = *g;
                    float3 b3 = f3(gb.x, gb.y, gb.z);
                    b3 *= (ld3(kp.albedo) * Cd * density_color / ld3(kp.extinction)) * float(kp.energy_inject);
                    *g = make_float4(b3.x, b3.y, b3.z, gb.w);
                } else {
                    float3 b3 = f3(beta[0], beta[beta_stride], beta[2 * beta_stride]);
                    b3 *= (ld3(kp.albedo) * Cd * density_color / ld3(kp.extinction)) * float(kp.energy_inject);
                    beta[0] = b3.x; beta[beta_stride] = b3.y; beta[2 * beta_stride] = b3.z;
                }
            } else {
                // instanced / emissive scenes: the per-leaf colour look-ups are deferred to scatter_event() in the service round, where
                // many rays run them at once instead of one or two lanes of a stepping warp (faster on the fireball)
                st.trv = density;                                   // free during a delta walk (the ratio walk re-initialises it)
                st.aux.x = __int_as_float(leaf);                    // aux is free during a delta walk, too
            }
            st.op = OP_GLUE; st.exit_reason = EX_SCATTER;
        }
    } else {
        st.trv = pmul(st.trv, pfma(-tc.sigma_r_inv, psub(density, tc.sigma_c), 1.0f));   // 1 - (rho - sigma_c) * sigma_r_inv, fused as in the reference SASS
        if (length(f3(st.trv)) < VPT_EPS) { st.op = OP_GLUE; st.exit_reason = EX_TR_DONE; }
    }
}

// The throughput factor of an accepted collision: albedo * Cd * density_colour / extinction * energy_inject (reference `sample`,
// render_kernel.cu:1664-1675).  Cd is the leaf's colour at the collision point -- the leaf located at the step's START, as the reference
// does -- and the colour LUT is indexed by density / sigma_max; the reference evaluates both at every step and drops them unless accepted.
VPT_DEV void scatter_event(PathState& st, const FrameShared& fs, const FrameArgs& fa, const TraceConsts& tc)
{
    const vpt_kernel_params& kp = fa.kp;
    const float density = st.trv;
    const float3 Cd = leaf_color(fs.sc, fs.vol0, __float_as_int(st.aux.x), st.wpos);
    const int index = int(floorf(fminf(fmaxf((density * tc.inv_max * 255.0f / kp.emission_pivot), 0.0f), 255.0f)));
    const float3 density_color = reinterpret_cast<const float3*>(kp.density_color_texture)[index];
    st.beta *= (ld3(kp.albedo) * Cd * density_color / ld3(kp.extinction)) * float(kp.energy_inject);
}

// ---- OP_TRBEGIN: reference Tr prologue (:1150-1167); the walk starts from (st.wpos, st.wdir) -----------------
VPT_DEV void begin_ratio_walk(PathState& st, const FrameShared& fs, const TraceConsts& tc, const SphereRec& sph)
{
    const SceneTables& sc = fs.sc;
    float3 p = st.wpos; const float3 d = st.wdir;
    float t_min, t_max, geo_dist = .0f, distance = .0f;
    st.op = OP_GLUE;                                            // unless a walk is really needed
    st.T_c = 1.0f;
    if (!aabb_contains(sc.root_pmin, sc.root_pmax, p)) {
        if (aabb_intersect(sc.root_pmin, sc.root_pmax, p, d, t_min, t_max)) p = madd3(p, d, padd(t_min, VPT_EPS));
        else { st.trv = 1.0f; return; }                         // misses the volume box: transmittance 1
    }
    aabb_intersect(sc.root_pmin, sc.root_pmax, p, d, t_min, distance);
    st.sphere_free = line_misses_sphere(sph, p, d);
    if (!st.sphere_free && sphere_intersect(sph, p, d, geo_dist, t_max)) { st.trv = 0.0f; return; }   // sphere occludes: BLACK
    st.T_c = expf(-tc.sigma_c * distance);
    st.wpos = p; st.t = 0.0f; st.distance = distance; st.trv = 1.0f;
    st.mode = W_RATIO; st.op = OP_STEP;
}

VPT_DEV float finish_ratio_walk(const PathState& st) { return clampf(st.trv * st.T_c, .0f, 1.0f); }

// ---- the integrator's control flow between heavy operations -------------------------------------------------
// kGroups (generic instantiation only): every L += also goes to the ray's light-group sums in lg->planes.  Mattes (the pack `mt`, one
// MatteIds pointer or empty): the id of the camera ray's first collision goes to the id plane (a lean kernel's volume is instance 0)
template <bool kLean, bool kGroups = false, class... Mt>
VPT_DEV void advance(PathState& st, const FrameShared& fs, const FrameArgs& fa, const TraceConsts& tc, const SphereRec& sph,
                     const LightGroups* lg = nullptr, const Mt*... mt)
{
    const SceneTables& sc = fs.sc;
    const vpt_kernel_params& kp = fa.kp;

    for (;;) {
        switch (st.phase) {
        case PH_BOUNCE_TOP:
            if (st.rd > kp.ray_depth) { st.op = OP_FINISH; return; }
            if (!st.have_closest) { st.op = OP_CLOSEST; st.phase = PH_TOP_HAVE; return; }
            st.phase = PH_TOP_HAVE;
            break;
        case PH_TOP_HAVE:
            if (st.first_walk && st.obj_c != 1) {                   // depth pass without a volume walk (:1883-1888)
                if (st.obj_c == 2) {
                    st.depth = length(st.org - (st.pos + st.dir * st.tmin_c));
                    if constexpr (sizeof...(Mt) > 0) matte_ids(mt...)->id[group_slot(st, fa)] = kMatteSphereId;
                }
                st.first_walk = false;
            }
            if (st.obj_c == 0) { st.op = OP_FINISH; return; }       // nothing ahead: every later bounce is a no-op
            if (st.obj_c == 1) {
                st.pos = madd3(st.pos, st.dir, padd(st.tmin_c, VPT_EPS));
                st.have_closest = false;
                st.vd = 1;
                st.phase = PH_VOL_ITER;
            } else st.phase = PH_SPHERE;                            // (a) and (b) see the same ray
            break;
        case PH_VOL_ITER:
            if (st.vd > kp.volume_depth) { st.phase = PH_VOL_DONE; break; }
            st.mi = false;
            st.wpos = st.pos; st.wdir = st.dir;
            if (!aabb_contains(sc.root_pmin, sc.root_pmax, st.pos)) {
                // `sample` leaves at once, and so does every remaining volume_depth iteration (ray unchanged, no draw)
                st.exit_reason = EX_OUTSIDE; st.vd = kp.volume_depth; st.phase = PH_AFTER_DELTA;
                break;
            }
            st.sphere_free = line_misses_sphere(sph, st.pos, st.dir);
            st.t = 0.0f; st.distance = .0f; st.mode = W_DELTA; st.op = OP_STEP; st.phase = PH_AFTER_DELTA;
            return;
        case PH_AFTER_DELTA: {
            st.pos = st.wpos;                                       // `sample` advances the caller's ray_pos
            int obj = 1;
            if (st.exit_reason == EX_SCATTER) { if (!kLean) scatter_event(st, fs, fa, tc); st.mi = true; }
            if (st.exit_reason == EX_DISTANCE) obj = 2;             // compiled reference: obj = 2 on every distance exit (Q4)
            if (st.first_walk) {
                st.depth = st.mi ? length(st.org - st.pos) : .0f;
                if constexpr (sizeof...(Mt) > 0) {
                    if (st.mi) matte_ids(mt...)->id[group_slot(st, fa)] = kLean ? 0u : collision_instance(sc, __float_as_int(st.aux.x), st.pos, last_draw(st.rng), tc.inv_max);
                }
                // the reference runs this identical walk twice (depth pass + integrator) and accumulates `tr` in
                // both; the replay adds the same densities again while tr < 1
                if (st.alpha < 1.0f) st.alpha += st.alpha;
                st.first_walk = false;
            }
            if (is_black(st.beta) || obj == 2) { st.phase = PH_VOL_DONE; break; }
            if (st.mi) hg_sample(st.dir, st.rng, kp.phase_g1);
            st.vd++; st.phase = PH_VOL_ITER;
            break;
        }
        case PH_AFTER_HG:
            st.vd++; st.phase = PH_VOL_ITER;
            break;
        case PH_VOL_DONE:
            if (st.mi) {
                st.tr_kind = TR_SUN; st.wpos = st.pos; st.wdir = tc.sun_dir;
                st.op = OP_TRBEGIN; st.phase = PH_AFTER_TR;
                return;
            }
            st.phase = PH_EMISSION;
            break;
        case PH_AFTER_TR: {
            const float tr = finish_ratio_walk(st);
            if (st.tr_kind == TR_SUN) {                             // reference estimate_sun (:1478-1516)
                const float cos_theta = dot(st.dir, tc.sun_dir);
                const float phase_pdf = hg_phase(cos_theta, kp.phase_g1);
                const float3 Ld = f3(tr) * phase_pdf;
                if constexpr (kGroups) {
                    const float3 t = Ld * ld3(kp.sun_color) * kp.sun_mult;
                    st.L = pfma3(t, st.beta, st.L);
                    group_fma(lg, group_slot(st, fa), LG_SUN, t, st.beta);
                } else st.L += Ld * ld3(kp.sun_color) * kp.sun_mult * st.beta;
                if (!kLean && fa.lights.num_lights > 0) { st.aux = f3(.0f); st.light_budget = 10; st.phase = PH_POINT_NEXT; }
                else st.phase = PH_EMISSION;
            } else if (!kLean && st.tr_kind == TR_POINT) {                    // reference point_light::Le, light.h:104-121
                if (st.light_budget < (int)fa.lights.num_lights) {
                    const vpt_point_light& pl = reinterpret_cast<const vpt_point_light*>(fa.lights.light_ptr)[st.light_index];
                    const float3 lpos = ld3(pl.pos);
                    const float3 wi = normalize(lpos - st.pos);
                    const float cos_theta = dot(st.dir, wi);
                    const float phase_pdf = hg_phase(cos_theta, kp.phase_g1);
                    const float sqr_dist = length(lpos * lpos - st.pos * st.pos);
                    const float falloff = 1 / sqr_dist;
                    st.aux += ld3(pl.color) * pl.power * f3(tr) * phase_pdf * falloff;
                }
                st.light_budget--;
                st.phase = PH_POINT_NEXT;
            } else {                                                // sphere branch tail (:1831-1833)
                if constexpr (kGroups) {
                    const float3 t = ld3(kp.sun_color) * kp.sun_mult * f3(tr) * fmaxf(dot(tc.sun_dir, st.aux), .0f);
                    st.L = pfma3(t, st.beta, st.L);
                    group_fma(lg, group_slot(st, fa), LG_SUN, t, st.beta);
                } else st.L += ld3(kp.sun_color) * kp.sun_mult * f3(tr) * fmaxf(dot(tc.sun_dir, st.aux), .0f) * st.beta;
                if (fa.planeD) fa.planeD[(size_t)st.pass * fa.geom.n_local + ray_local_pixel(fa.geom, st.lp)] = make_float4(st.pos.x, st.pos.y, st.pos.z, 0.f);   // env_pos = ray_pos
                st.sphere_bounced = true;
                st.rd++; st.have_closest = false;
                st.phase = PH_BOUNCE_TOP;
            }
            break;
        }
        case PH_POINT_NEXT: {                                       // reference estimate_point_light (:1445-1475)
            if (kLean) { st.phase = PH_EMISSION; break; }
            if (st.light_budget < 0) {
                if constexpr (kGroups) { st.L = pfma3(st.aux, st.beta, st.L); group_fma(lg, group_slot(st, fa), LG_POINT, st.aux, st.beta); }
                else st.L += st.aux * st.beta;
                st.phase = PH_EMISSION; break;
            }
            const vpt_point_light* lp = reinterpret_cast<const vpt_point_light*>(fa.lights.light_ptr);
            st.light_index = int(floorf(st.rng.next() * fa.lights.num_lights));
            st.tr_kind = TR_POINT; st.wpos = st.pos; st.wdir = normalize(ld3(lp[st.light_index].pos) - st.pos);
            st.op = OP_TRBEGIN; st.phase = PH_AFTER_TR;
            return;
        }
        case PH_EMISSION:
            if (!kLean && kp.emission_scale > 0 && st.mi) {
                st.wpos = st.pos; st.wdir = st.dir; st.t = 0.0f; st.aux = f3(.0f);
                st.mode = W_EMIT; st.op = OP_STEP; st.phase = PH_AFTER_EMIT;
                return;
            }
            st.phase = PH_AFTER_VOLUME;
            break;
        case PH_AFTER_EMIT:
            st.L += st.aux;
            if constexpr (kGroups) group_add(lg, group_slot(st, fa), LG_EMISSION, st.aux);
            st.phase = PH_AFTER_VOLUME;
            break;
        case PH_AFTER_VOLUME: {                                     // the ray moved since the last test
            // Later bounces cannot change the sample unless the sphere comes into play (quirk Q21: a ray inside the box is
            // teleported to its exit, a ray outside it and leaving sees nothing).  If this ray's line provably misses the
            // sphere and the position is not exactly on the box boundary, retire the path here: bit-identical output.
            const bool inside_strict = st.pos.x > sc.root_pmin[0] && st.pos.x < sc.root_pmax[0] && st.pos.y > sc.root_pmin[1] &&
                                       st.pos.y < sc.root_pmax[1] && st.pos.z > sc.root_pmin[2] && st.pos.z < sc.root_pmax[2];
            const bool outside = !aabb_contains(sc.root_pmin, sc.root_pmax, st.pos);
            // outside here means the walk stepped out of the box along dir (or never re-entered it): the box lies behind
            if ((inside_strict || (outside && st.exit_reason == EX_OUTSIDE && !st.sphere_bounced)) && line_misses_sphere(sph, st.pos, st.dir)) { st.op = OP_FINISH; return; }
            st.op = OP_CLOSEST; st.phase = PH_AFTERVOL_HAVE;
            return;
        }
        case PH_AFTERVOL_HAVE:
            if (st.obj_c == 2) { st.phase = PH_SPHERE; break; }
            st.rd++; st.phase = PH_BOUNCE_TOP;                      // next bounce starts from the same ray: reuse the test
            break;
        case PH_SPHERE: {                                           // bounce off the reference sphere (:1807-1834)
            st.pos += st.dir * st.tmin_c;
            const float3 normal = normalize((st.pos - sph.center) / sph.radius);
            const float3 nl = dot(normal, st.dir) < 0 ? normal : normal * -1;
            const float phi = 2 * VPT_PI_F * st.rng.next();
            const float r2 = st.rng.next();
            const float r2s = sqrtf(r2);
            const float3 w = normalize(nl);
            const float3 u = normalize(cross((fabs(w.x) > .1 ? f3(0, 1, 0) : f3(1, 0, 0)), w));
            const float3 v = cross(w, u);
            const float3 hemisphere_dir = normalize(u * cosf(phi) * r2s + v * sinf(phi) * r2s + w * sqrtf(1 - r2));
            const float3 ref = reflect3(st.dir, nl);
            st.dir = lerp3(ref, hemisphere_dir, sph.roughness);
            st.pos += normal * VPT_EPS;
            st.beta *= sph.color;
            st.aux = normal;
            st.tr_kind = TR_SPHERE; st.wpos = st.pos; st.wdir = tc.sun_dir;
            st.op = OP_TRBEGIN; st.phase = PH_AFTER_TR;
            return;
        }
        default:
            st.op = OP_FINISH;
            return;
        }
    }
}

#include "vpt_trace_vol.cuh"

// A path from queue record `slot` (k_generate): camera ray, pixel, pass, the draw count of the lens sampler in rng.k (the caller seeds the
// stream), and k_generate's closest-object test.  A prestepped record is a delta walker at the walk start k_generate found.
template <int kInteg>
VPT_DEV void start_path(PathState& st, const FrameArgs& fa, uint32_t slot)
{
    const float4 r0 = __ldg(fa.queue_dir + slot);
    const uint2 id = __ldg(fa.queue_id + slot);
    st.dir = f3(r0.x, r0.y, r0.z);
    st.qslot = slot;
    st.org = ray_origin(fa, slot);
    st.lp = id.x; st.pass = id.y & 63u;
    st.rng.k = (id.y >> 6) & 1023u;
    reset_path(st);
    st.tmin_c = r0.w; st.obj_c = (int)((id.y >> 16) & 3u); st.have_closest = true;       // k_generate already ran the first test
    st.phase = kInteg ? (int)VP_START : (int)PH_BOUNCE_TOP; st.op = OP_GLUE;
    if ((id.y >> 18) & 1u) {
        // k_generate already hopped over the empty nodes in front of this ray: it is a delta walker at `wpos`
        const float4 ws = __ldg(fa.queue_aux + slot);
        st.wpos = f3(ws.x, ws.y, ws.z); st.pos = st.wpos;
        st.have_closest = false; st.sphere_free = true;
        st.phase = kInteg ? (int)VP_AFTER_DELTA : (int)PH_AFTER_DELTA; st.op = OP_STEP;
    }
}

// kLean: the instantiation may write compact records (the host allocates them for the lean kernels only, see frame_setup)
template <int kInteg, bool kLean>
VPT_DEV void write_sample(const PathState& st, const FrameArgs& fa)
{
    uint32_t lp = st.lp;
    if (fa.geom.n_ranks > 1) lp = ray_local_pixel(fa.geom, st.lp);
    const size_t o = (size_t)st.pass * fa.geom.n_local + lp;
    if (kLean && !fa.planeB) {
        // compact record (HDRI environment): the finished radiance, so k_resolve<0> reads one float4 per sample; tr only reaches raw.w
        // from the chunk's last pass.  A depth is never the sentinel: arithmetic NaNs are 0x7fffffff.
        const float3 v = hdri_radiance((cudaTextureObject_t)fa.kp.env_tex, ld3(fa.kp.sky_color), st.dir, st.L, st.beta);
        fa.planeA[o] = make_float4(v.x, v.y, v.z, st.depth);
        if (st.pass == (uint32_t)fa.n_passes - 1u) fa.plane_tr[lp] = st.alpha;
        return;
    }
    fa.planeA[o] = make_float4(st.dir.x, st.dir.y, st.dir.z, st.alpha);                 // final direction, tr
    fa.planeB[o] = make_float4(st.L.x, st.L.y, st.L.z, st.depth);                       // L, depth
    fa.planeC[o] = make_float4(st.beta.x, st.beta.y, st.beta.z, 1.f);                   // beta
    if (kInteg) {
        // vol_integrator evaluates the sky from env_pos while the throughput is still ~white, else from where the path ended (:1750)
        float3 e = length(st.beta) > 0.9999f ? st.org : st.pos;
        if (fa.debug_flags & 16) e = st.org;                                                // development probes
        if (fa.debug_flags & 32) e = st.pos;
        fa.planeD[o] = make_float4(e.x, e.y, e.z, 0.f);
    } else if (fa.planeD && !st.sphere_bounced) fa.planeD[o] = make_float4(st.org.x, st.org.y, st.org.z, 0.f);   // env_pos = camera origin unless the sphere branch moved it
}

// kInteg = 0: direct integrator (the tuned headline path); kInteg = 1: volumetric path integrator, which additionally needs the
// caller's AtmosphereParameters in the kernel (sky radiance decides whether a transmittance walk is run at all)
struct NoAtmo { int pad[4]; };

// kGroups (generic kernels): the light-group instantiation, which takes the LightGroups as one more argument (the pack `lgs`, empty
// otherwise), so the kernels without groups keep their parameter block.  The matte instantiations end the pack with a MatteIds; it is the
// pack, not a template flag, that selects them, so every kernel without mattes keeps its name as well.
template <class... Lg> constexpr bool has_matte_ids = (std::is_same<Lg, MatteIds>::value || ... || false);
template <int kInteg, bool kLean, int kSlots, bool kCells = false, bool kGroups = false, class... Lg>
__global__ void __launch_bounds__(trace_threads(kLean, kSlots, kCells), trace_min_ctas(kLean, kSlots, kCells))
k_trace(const FrameArgs fa, const typename std::conditional<kInteg != 0, vpt_atmosphere, NoAtmo>::type atm, const Lg... lgs)
{
    static_assert(sizeof...(Lg) == (kGroups ? 1 : 0) + (has_matte_ids<Lg...> ? 1 : 0),
                  "k_trace<..., true> takes one LightGroups, then a MatteIds for the mattes; the other instantiations only the MatteIds or none");
    static_assert(!kGroups || !kLean, "lean kernels keep their light groups in the wide records (L is the sun group)");
    static_assert(!has_matte_ids<Lg...> || !kCells, "cell mode has no mattes");
    // (the LightGroups are reached through lg_of(lgs...) where they are used: a pointer variable in every instantiation, even unused,
    // moved two stack stores of k_trace<1, false, 3>)
    __shared__ FrameShared fs;
    extern __shared__ float pool_smem[];                         // warps x kWords x kPool words (opt-in dynamic shared memory)
    __shared__ EmptyAhead ea;
    // the lean kernels end walks at "empty ahead" (the render call's table, staged with the octree); the generic ones keep their hot loop
    // as it was (on the fireball, config 3, the extra code of the shortcut cost more in the fetch-bound loop than its hops saved)
    load_frame_shared(fs, fa.scene, kLean ? &ea : nullptr);
    const SceneTables& sc = fs.sc;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned lt_mask = (1u << lane) - 1u;

    const TraceConsts tc = make_trace_consts(sc, fa.kp);
    const SphereRec sph = load_sphere(fa.sphere);

    constexpr int kPool = 32 * kSlots;
    constexpr bool kGroups16 = kLean && kSlots == 3;             // the headline kernels park their rays in 16-byte groups
    constexpr bool kLean28 = kLean && kSlots == 2;               // ... the lean ones at 2 rays per lane in 29 words
    constexpr int kWords = kLean28 ? kLeanRayWords : kRayWords;
    typename std::conditional<kGroups16, PoolGroups<kSlots>, typename std::conditional<kLean28, PoolLean<kPool>, PoolView<kPool>>::type>::type pv;
    float* const pool_warp = pool_smem + (size_t)warp * kWords * kPool;   // this warp's kWords * kPool words
    if constexpr (kGroups16) {
        pv.q = reinterpret_cast<float4*>(pool_warp) + lane;
        pv.h = reinterpret_cast<float2*>(pool_warp + kRayGroups4 * 4 * kPool) + lane;
    } else pv.w = pool_warp + lane;
    if constexpr (kLean28) { pv.sun_dir = tc.sun_dir; pv.sigma_c = tc.sigma_c; }
    constexpr int OP_NOSLOT = 15;                                 // third slot disabled when kSlots == 2
    int tag0 = OP_IDLE, tag1 = OP_IDLE, tag2 = (kSlots > 2) ? OP_IDLE : OP_NOSLOT;   // operation each of my rays waits for

    const unsigned q_count = *fa.queue_count;
    bool queue_dry = (q_count == 0);
    uint32_t nlook = 0, lane_steps = 0, warp_iters = 0, lane_ops = 0, warp_ops = 0, lane_rays = 0;   // statistics
    HopStats hs = {0u, 0u, 0u, 0u};
    PathState st;

    for (;;) {
        // ---- refill free slots from the global queue: one atomic per warp, one record per lane that has room ----------
        const bool has_idle = (tag0 == OP_IDLE) | (tag1 == OP_IDLE) | (tag2 == OP_IDLE);
        const unsigned idle_lanes = __ballot_sync(0xffffffffu, has_idle);
        if (!queue_dry && __popc(idle_lanes) >= fa.sched_min_lanes) {
            unsigned base = 0;
            const int leader = __ffs(idle_lanes) - 1;
            if (lane == leader) base = atomicAdd(fa.queue_head, (unsigned)__popc(idle_lanes));
            base = __shfl_sync(0xffffffffu, base, leader);
            if (base + __popc(idle_lanes) >= q_count) queue_dry = true;
            const unsigned slot = base + __popc(idle_lanes & lt_mask);
            if (has_idle && slot < q_count) {
                const int j = (tag0 == OP_IDLE) ? 0 : (tag1 == OP_IDLE) ? 1 : 2;
                start_path<kInteg>(st, fa, slot);
                if constexpr (kLean28) st.rng.key = ray_global_pixel(fa.geom, st.lp);   // the record keeps the stream's key
                if constexpr (kGroups) {                          // the sample slot's group sums start at 0 (integrator 0 keeps no environment sum)
                    const size_t s = group_slot(st, fa);
                    #pragma unroll
                    for (int k = 0; k < (kInteg ? 12 : 9); ++k) lg_of(lgs...)->planes[(size_t)k * lg_of(lgs...)->stride + s] = 0.0f;
                }
                store_ray(pv, j, st);
                if (j == 0) tag0 = st.op; else if (j == 1) tag1 = st.op; else tag2 = st.op;
                lane_rays++;
            }
        }

        // ---- vote: step, or service the rays that wait for bookkeeping / a closest-object test / a transmittance set-up? ----
        const bool has_step = (tag0 == OP_STEP) | (tag1 == OP_STEP) | (tag2 == OP_STEP);
        const bool svc0 = (tag0 != OP_STEP) & (tag0 != OP_IDLE), svc1 = (tag1 != OP_STEP) & (tag1 != OP_IDLE), svc2 = (tag2 != OP_STEP) & (tag2 != OP_IDLE) & (tag2 != OP_NOSLOT);
        const int nS = __popc(__ballot_sync(0xffffffffu, has_step));
        const int nV = __popc(__ballot_sync(0xffffffffu, svc0 | svc1 | svc2));
        if ((nS | nV) == 0) {
            if (queue_dry) break;                                  // nothing parked, nothing left to fetch
            continue;                                              // everything idle: the refill above takes records next round
        }

        if (nV > nS) {
            // ---- service round: one parked ray per participating lane runs [closest-object test] -> integrator control flow
            //      (incl. HG resampling, NEE bookkeeping, retirement) -> [transmittance set-up]; each block has one code site ----
            const int j = svc0 ? 0 : svc1 ? 1 : svc2 ? 2 : -1;
            if (j >= 0) {
                load_ray(pv, j, st, fa);
                st.op = (j == 0) ? tag0 : (j == 1) ? tag1 : tag2;
                if (st.op == OP_CLOSEST) {
                    st.obj_c = closest_object(sc, sph, st.pos, st.dir, st.tmin_c);
                    st.have_closest = true; st.op = OP_GLUE;
                }
                if (st.op == OP_GLUE) {
                    if constexpr (has_matte_ids<Lg...>) {
                        const LightGroups* lgp = nullptr;
                        if constexpr (kGroups) lgp = lg_of(lgs...);
                        if constexpr (kInteg != 0) advance_vol<kGroups>(st, fs, fa, atm, tc, sph, lgp, mt_of(lgs...));
                        else advance<kLean, kGroups>(st, fs, fa, tc, sph, lgp, mt_of(lgs...));
                    }
                    else if constexpr (kInteg != 0 && kGroups) advance_vol<true>(st, fs, fa, atm, tc, sph, lg_of(lgs...));
                    else if constexpr (kInteg != 0) advance_vol(st, fs, fa, atm, tc, sph);
                    else if constexpr (kGroups) advance<kLean, true>(st, fs, fa, tc, sph, lg_of(lgs...));
                    else advance<kLean>(st, fs, fa, tc, sph);
                }
                if (st.op == OP_TRBEGIN) begin_ratio_walk(st, fs, tc, sph);
                if (st.op == OP_FINISH) { write_sample<kInteg, kLean>(st, fa); st.op = OP_IDLE; }
                else store_ray(pv, j, st);
                if (j == 0) tag0 = st.op; else if (j == 1) tag1 = st.op; else tag2 = st.op;
                lane_ops++;
            }
            warp_ops++;
            continue;
        }

        // ---- stepping loop: a lane steps one of its walkers; when that walk ends it parks the ray and swaps in its next walker ----
        {
            int cur = -1;
            int parked_lanes = nV;                                // lanes with something to service (grows as walks end)
            for (;;) {
                if (cur < 0) {
                    cur = (tag0 == OP_STEP) ? 0 : (tag1 == OP_STEP) ? 1 : (tag2 == OP_STEP) ? 2 : -1;
                    if (cur >= 0) { load_walk(pv, cur, st, fa); st.op = OP_STEP; }
                }
                const unsigned walking = __ballot_sync(0xffffffffu, cur >= 0);
                if (walking == 0u) break;
                // few walkers left and a fuller group is waiting: park and let the vote pick it
                if (__popc(walking) < fa.sched_min_lanes && parked_lanes > __popc(walking)) {
                    if (cur >= 0) { store_walk(pv, cur, st); cur = -1; }
                    break;
                }
                if (cur >= 0) {
                    if constexpr (kGroups16) walk_step<kLean, kCells, kLean>(st, fs, fa, tc, sph, nlook, &pv.g(G_BETA, cur).x, 1, &ea, &hs);
                    else walk_step<kLean, kCells, kLean>(st, fs, fa, tc, sph, nlook, &pv.f(9, cur), kPool, &ea, &hs); lane_steps++;
                    if (st.op != OP_STEP) {                        // walk ended: park the ray with its new tag
                        store_walk(pv, cur, st);
                        if (cur == 0) tag0 = st.op; else if (cur == 1) tag1 = st.op; else tag2 = st.op;
                        cur = -1;
                    }
                }
                parked_lanes = __popc(__ballot_sync(0xffffffffu, ((tag0 != OP_STEP) & (tag0 != OP_IDLE)) | ((tag1 != OP_STEP) & (tag1 != OP_IDLE)) | ((tag2 != OP_STEP) & (tag2 != OP_IDLE) & (tag2 != OP_NOSLOT))));
                warp_iters++;
            }
        }
    }

    if (fa.counters) {                                        // optional statistics (one atomic set per warp)
        unsigned long long a = nlook, b = lane_steps, c = lane_ops, d = lane_rays;
        for (int o = 16; o > 0; o >>= 1) {
            a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); c += __shfl_xor_sync(0xffffffffu, c, o); d += __shfl_xor_sync(0xffffffffu, d, o);
        }
        if (lane == 0) {
            atomicAdd(fa.counters + 0, a); atomicAdd(fa.counters + 1, b); atomicAdd(fa.counters + 2, (unsigned long long)warp_iters);
            atomicAdd(fa.counters + 3, c); atomicAdd(fa.counters + 4, (unsigned long long)warp_ops); atomicAdd(fa.counters + 5, d);
        }
        if constexpr (kLean) {                                // hop statistics: counted by the kernels that end walks at "empty ahead"
            uint32_t h[4] = {hs.delta, hs.ratio, hs.emit, hs.ahead};
            #pragma unroll
            for (int k = 0; k < 4; ++k) {
                for (int o = 16; o > 0; o >>= 1) h[k] += __shfl_xor_sync(0xffffffffu, h[k], o);
                if (lane == 0) atomicAdd(fa.counters + 8 + k, (unsigned long long)h[k]);
            }
        }
    }
}
