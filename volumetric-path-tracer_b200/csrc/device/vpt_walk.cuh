// vpt_walk.cuh -- geometry tests, octree point location and the unified tracking step.
//
// One step of delta tracking (reference `sample`, render_kernel.cu:1556-1681), of residual-ratio
// tracking (`Tr`, :1138-1273) and of the emission walk (`estimate_emission`, :1275-1339) share
// everything except a few instructions: locate the position in the fixed depth-3 octree, skip an
// empty node, draw a free-flight distance against the root majorant, advance, look the density up.
// The wavefront trace kernel therefore runs ONE step body for all three kinds of walk so that the
// lanes of a warp stay converged whatever estimator their ray is in.
#pragma once
#include "vpt_math.cuh"
#include "vpt_scene.cuh"
#include "../../../include/vpt_abi.h"

namespace vpt {

// ---- shared-memory copy of the octree's internal levels ------------------------------------------
struct OctShared {
    OctInternal node[kOctInternalNodes];
};

VPT_DEV void stage_octree(OctShared& dst, const SceneTables& sc) {
    // 73 * 48 B = 3504 B, copied as 16-byte words by the whole CTA
    const uint4* src = reinterpret_cast<const uint4*>(sc.internal);
    uint4* d = reinterpret_cast<uint4*>(dst.node);
    for (int i = threadIdx.x; i < kOctInternalNodes * 3; i += blockDim.x) d[i] = __ldg(src + i);
}

// ---- AABB slab test (reference AABB::Intersect, bvh/AABB.h:182-205) ------------------------------
// Writes tmin/tmax exactly as the reference does (tmax is defined even when the test fails).
VPT_DEV bool aabb_intersect(const float pmin[3], const float pmax[3], float3 o, float3 d, float& tmin, float& tmax) {
    const float ix = 1.0f / d.x, iy = 1.0f / d.y, iz = 1.0f / d.z;
    const float t1 = (pmin[0] - o.x) * ix, t2 = (pmax[0] - o.x) * ix;
    const float t3 = (pmin[1] - o.y) * iy, t4 = (pmax[1] - o.y) * iy;
    const float t5 = (pmin[2] - o.z) * iz, t6 = (pmax[2] - o.z) * iz;
    tmin = fmaxf(fmaxf(fminf(t1, t2), fminf(t3, t4)), fminf(t5, t6));
    tmax = fminf(fminf(fmaxf(t1, t2), fmaxf(t3, t4)), fmaxf(t5, t6));
    if (tmax <= 0.0f) return false;
    if (tmin > tmax) return false;
    if (tmin < 0) {
        tmin = tmax;
        if (tmin < 0) return false;
    }
    return true;
}

VPT_DEV bool aabb_contains(const float pmin[3], const float pmax[3], float3 p) {
    return p.x >= pmin[0] && p.x <= pmax[0] && p.y >= pmin[1] && p.y <= pmax[1] && p.z >= pmin[2] && p.z <= pmax[2];
}

// ---- sphere (reference sphere::intersect + find_discr, geometry/geometry.h:46-70, 114-137) -------
struct SphereRec { float3 center; float radius; float3 color; float roughness; };

VPT_DEV bool solve_quadratic(float a, float b, float c, float& x1, float& x2) {
    if (b == 0) {
        if (a == 0) return false;
        x1 = 0; x2 = sqrtf(-c / a);
        return true;
    }
    float discr = pfma(b, b, pmul(pmul(a, -4.0f), c));         // b*b - 4*a*c as the reference build evaluates it
    if (discr < 0) return false;
    float q = (b < 0.f) ? -0.5f * (b - sqrtf(discr)) : -0.5f * (b + sqrtf(discr));
    x1 = q / a;
    x2 = c / q;
    return true;
}

VPT_DEV bool sphere_intersect(const SphereRec& s, float3 ray_pos, float3 ray_dir, float& t_min, float& t_max) {
    float3 orig = ray_pos - s.center;
    float A = dot(ray_dir, ray_dir);
    float Bh = dot(ray_dir, orig);
    float B = padd(Bh, Bh);
    float C = psub(dot(orig, orig), pmul(s.radius, s.radius));
    if (!solve_quadratic(A, B, C, t_min, t_max)) return false;
    if (t_min > t_max) { float tmp = t_max; t_max = t_min; t_min = tmp; }
    if (t_min < 0) {
        t_min = t_max;
        if (t_min < 0) return false;
    }
    return true;
}

// Conservative test: true only if the infinite line p + s*d stays clear of the sphere enlarged by a margin three orders
// of magnitude above float rounding (2e-3 of |c-p|^2 plus 2 % of r^2).  Then every sphere::intersect the reference
// evaluates along this line returns "no hit" whatever the rounding, so those tests (and whatever only they could
// trigger) are skipped; lines that come anywhere near the sphere take the exact path.
VPT_DEV bool line_misses_sphere(const SphereRec& s, float3 p, float3 d)
{
    const float3 oc = s.center - p;
    const float oc2 = oc.x * oc.x + oc.y * oc.y + oc.z * oc.z, dd = d.x * d.x + d.y * d.y + d.z * d.z, b = oc.x * d.x + oc.y * d.y + oc.z * d.z;
    const float dist2 = oc2 - b * b / dd;
    return dist2 > 1.02f * s.radius * s.radius + 2e-3f * oc2 + 1e-6f;
}

// Nearest of {octree root box, reference sphere}: 1 = volume box, 2 = sphere, 0 = neither
// (reference get_closest_object, render_kernel.cu:1118-1135).
VPT_DEV int closest_object(const SceneTables& sc, const SphereRec& sph, float3 ray_pos, float3 ray_dir, float& t_min) {
    float tmin1 = VPT_M_INF, tmax1 = -VPT_M_INF, tmin2 = VPT_M_INF, tmax2 = -VPT_M_INF;
    bool i1 = aabb_intersect(sc.root_pmin, sc.root_pmax, ray_pos, ray_dir, tmin1, tmax1);
    bool i2 = sphere_intersect(sph, ray_pos, ray_dir, tmin2, tmax2);
    if (i1 && !i2) { t_min = tmin1; return 1; }
    if (!i1 && i2) { t_min = tmin2; return 2; }
    if (i1 && i2) {
        if (tmin1 < tmin2) { t_min = tmin1; return 1; }
        if (tmin2 < tmin1) { t_min = tmin2; return 2; }
    }
    return 0;
}

// ---- octree point location ------------------------------------------------------------------------
// The reference scans children 0..7 and takes the FIRST whose inclusive box contains the point
// (render_kernel.cu:1102-1115); with the child order of divide_bbox (bvh_kernels.cu:150-202) that
// is exactly: x- unless p.x > half.x, y+ unless p.y < half.y, z- unless p.z > half.z
// (SURVEY 8(a-O)).  Child boxes reuse the parent's pmin/half/pmax floats, so comparing against the
// parent's three split planes gives bit-identical leaf indices.
VPT_DEV int oct_child(const OctInternal& n, float3 p) {
    const int xplus = !(p.x <= n.half[0]);
    const int yminus = !(p.y >= n.half[1]);
    const int zplus = !(p.z <= n.half[2]);
    return xplus + 2 * yminus + 4 * zplus;
}

// Exit distance of child `c` of node `n` for the empty-space skip: tmax of the slab test on the
// child's box (the reference ignores the hit/miss result, render_kernel.cu:1613-1615).
VPT_DEV float oct_child_exit(const OctInternal& n, int c, float3 o, float3 d) {
    float cmin[3], cmax[3];
    const bool xp = c & 1, ym = c & 2, zp = c & 4;
    cmin[0] = xp ? n.half[0] : n.pmin[0];  cmax[0] = xp ? n.pmax[0] : n.half[0];
    cmin[1] = ym ? n.pmin[1] : n.half[1];  cmax[1] = ym ? n.half[1] : n.pmax[1];
    cmin[2] = zp ? n.half[2] : n.pmin[2];  cmax[2] = zp ? n.pmax[2] : n.half[2];
    float tmin, tmax;
    aabb_intersect(cmin, cmax, o, d, tmin, tmax);
    return tmax;
}

// ---- "nothing populated ahead": the orthant occupancy table (DESIGN.md section 8j) -----------------------------------------------
// A walk only moves forward: every move is p += d * t with t >= 0, so along each axis no coordinate ever moves against the sign of d.
// Read the octree as an 8x8x8 grid of cells, the cell coordinate on an axis being the three "upper side" bits of the descent (x: p.x >
// half.x, y: p.y >= half.y, z: p.z > half.z, levels 1, 2, 3 from the top).  Each bit is monotone in its coordinate, and two points
// whose descents share a prefix on an axis are compared against the same split plane at the next level -- provided every non-empty
// node with that prefix splits the axis at the same float, which build_empty_ahead checks.  So the cell coordinate is monotone too:
// from any point in an empty node N, every later position of the walk lies in a cell of N's block or beyond it in the direction of d
// (the orthant of N's block for the octant of d).  If no populated leaf lies there, the walk only hops over empty nodes until it
// leaves the root box.  The table holds that answer for every (node, child) pair below the root and every octant: integer-only and
// conservative, no float margin.
// (kAheadEntries and EmptyAhead: vpt_scene.cuh)
struct AheadScratch {
    unsigned long long occ[8];                    // [z] populated leaves, bit y * 8 + x (cell coordinates)
    unsigned long long sfx[8][8];                 // [octant][z] cells whose orthant holds a populated leaf
    int bad;                                      // the split planes do not form one grid: every entry stays "maybe"
};

// octant of a direction: bit 0 x < 0, bit 1 y < 0, bit 2 z < 0 (a zero component may take either side: it never moves)
VPT_DEV int dir_octant(float3 d) { return (d.x < 0.0f ? 1 : 0) | (d.y < 0.0f ? 2 : 0) | (d.z < 0.0f ? 4 : 0); }
VPT_DEV bool empty_ahead(const EmptyAhead& ea, int entry, float3 d) { return (ea.bit[entry] >> dir_octant(d)) & 1u; }

// upper-side bit of child c on axis a (y is reversed in the child order: bit 1 set means y-minus)
VPT_DEV int child_upper(int c, int a) { return a == 1 ? ((c >> 1) & 1) ^ 1 : (c >> (a == 0 ? 0 : 2)) & 1; }

// Built by the whole CTA from the staged internal nodes (`oct` must be complete; ends with a barrier), once per render call by
// k_empty_ahead.  enable == false leaves every entry 0: the walks then hop exactly as without the table.
VPT_DEV void build_empty_ahead(EmptyAhead& ea, AheadScratch& s, const OctShared& oct, bool enable)
{
    const int t = threadIdx.y * blockDim.x + threadIdx.x, nt = blockDim.x * blockDim.y;
    const uint32_t re = oct.node[0].child_empty;
    auto node_full = [&](int i) {                  // internal node i (1..72) holds a volume
        if (i < 9) return !((re >> (i - 1)) & 1u);
        const int c1 = (i - 9) >> 3, c2 = (i - 9) & 7;
        return !((re >> c1) & 1u) && !((oct.node[1 + c1].child_empty >> c2) & 1u);
    };
    if (t == 0) s.bad = enable ? 0 : 1;
    __syncthreads();
    // (1) every non-empty node splits an axis at the same float as the non-empty nodes of its level that share its cell prefix on that
    //     axis (their children differ only in the other two axes' bits)
    int bad = 0;
    for (int i = 1 + t; i < kOctInternalNodes; i += nt) {
        if (!node_full(i)) continue;
        const bool l1 = i < 9;
        const int c1 = l1 ? i - 1 : (i - 9) >> 3, c2 = l1 ? 0 : (i - 9) & 7;
        for (int a = 0; a < 3; ++a) {
            const int free_bits = 7 & ~(1 << a);
            for (int m1 = 0; m1 < 8; ++m1) for (int m2 = 0; m2 < (l1 ? 1 : 8); ++m2) {
                if ((m1 & ~free_bits) || (m2 & ~free_bits) || (m1 | m2) == 0) continue;
                const int j = l1 ? 1 + (c1 ^ m1) : 9 + (c1 ^ m1) * 8 + (c2 ^ m2);
                if (node_full(j) && !(oct.node[j].half[a] == oct.node[i].half[a])) bad = 1;
            }
        }
    }
    if (bad) s.bad = 1;
    // (2) populated leaves, one (y, z) row of cells per thread
    for (int r = t; r < 64; r += nt) {
        const int iy = r & 7, iz = r >> 3;
        uint32_t row = 0;
        for (int ix = 0; ix < 8; ++ix) {
            auto child = [&](int b) { return ((ix >> b) & 1) | ((((iy >> b) & 1) ^ 1) << 1) | (((iz >> b) & 1) << 2); };
            const int c1 = child(2), c2 = child(1), c3 = child(0);
            const bool full = !((re >> c1) & 1u) && !((oct.node[1 + c1].child_empty >> c2) & 1u) &&
                              !((oct.node[9 + c1 * 8 + c2].child_empty >> c3) & 1u);
            row |= (uint32_t)full << ix;
        }
        reinterpret_cast<uint8_t*>(s.occ)[r] = (uint8_t)row;
    }
    __syncthreads();
    // (3) per octant, the cells from which a populated leaf lies ahead: OR over z in the direction of travel, then suffix-OR sweeps in x
    //     (within each byte) and y (across bytes)
    for (int k = t; k < 64; k += nt) {
        const int o = k >> 3, iz = k & 7;
        unsigned long long p = 0;
        for (int z = 0; z < 8; ++z) if ((o & 4) ? z <= iz : z >= iz) p |= s.occ[z];
        if (o & 1) { p |= (p << 1) & 0xfefefefefefefefeull; p |= (p << 2) & 0xfcfcfcfcfcfcfcfcull; p |= (p << 4) & 0xf0f0f0f0f0f0f0f0ull; }
        else       { p |= (p >> 1) & 0x7f7f7f7f7f7f7f7full; p |= (p >> 2) & 0x3f3f3f3f3f3f3f3full; p |= (p >> 4) & 0x0f0f0f0f0f0f0f0full; }
        if (o & 2) { p |= p << 8; p |= p << 16; p |= p << 32; }
        else       { p |= p >> 8; p |= p >> 16; p |= p >> 32; }
        s.sfx[o][iz] = p;
    }
    __syncthreads();
    // (4) each entry's block corner that comes first along the octant's direction; its bit answers for the whole block
    for (int e = t; e < kAheadEntries + 8; e += nt) {
        uint32_t v = 0;
        if (e < kAheadEntries && !s.bad) {
            const int lvl = e < 8 ? 1 : e < 72 ? 2 : 3;
            const int j = lvl == 1 ? e : lvl == 2 ? e - 8 : e - 72;
            const int cs[3] = {lvl == 1 ? j : lvl == 2 ? j >> 3 : j >> 6, lvl == 2 ? j & 7 : (j >> 3) & 7, j & 7};
            const int size = 8 >> lvl;
            int lo[3];
            for (int a = 0; a < 3; ++a) {
                lo[a] = 0;
                for (int l = 0; l < lvl; ++l) lo[a] += child_upper(cs[l], a) << (2 - l);
            }
            for (int o = 0; o < 8; ++o) {
                const int cx = (o & 1) ? lo[0] + size - 1 : lo[0];
                const int cy = (o & 2) ? lo[1] + size - 1 : lo[1];
                const int cz = (o & 4) ? lo[2] + size - 1 : lo[2];
                if (!((s.sfx[o][cz] >> (cy * 8 + cx)) & 1ull)) v |= 1u << o;
            }
        }
        ea.bit[e] = (uint8_t)v;
    }
    __syncthreads();
}

// Returns leaf index 0..511, or -1 "outside the root box", or -2 "skipped an empty node" (ray_pos advanced).
// kOneExit: one code site for the empty-child exit instead of one per level -- 64 instructions shorter; faster in k_generate
// and slightly slower in the trace kernel's stepping loop, so each caller picks its form.  Same arithmetic either way.
// kAhead: at an empty node whose entry in `ea` says no populated leaf lies ahead (and `allow`), return -3 "empty ahead" instead of
// hopping: the hops would only carry ray_pos out of the root box, drawing nothing.  ray_pos is then left where it was.
template <bool kOneExit = false, bool kAhead = false>
VPT_DEV int oct_locate_or_skip(const OctShared& oct, const SceneTables& sc, float3& ray_pos, float3 ray_dir,
                               const EmptyAhead* ea = nullptr, bool allow = true) {
    if (!aabb_contains(sc.root_pmin, sc.root_pmax, ray_pos)) return -1;
    if (kOneExit) {
    // three levels of descent, ONE code site for the empty-child exit (the slab test of the child box is the bulky part)
    const OctInternal* n = &oct.node[0];
    int c = oct_child(*n, ray_pos);
    int leaf = c * 64;
    int entry = c;
    bool empty = (n->child_empty >> c) & 1u;
    if (!empty) {
        const int c1 = c;
        n = &oct.node[1 + c1];
        c = oct_child(*n, ray_pos);
        leaf += c * 8;
        if (kAhead) entry = 8 + leaf / 8;
        empty = (n->child_empty >> c) & 1u;
        if (!empty) {
            n = &oct.node[9 + c1 * 8 + c];
            c = oct_child(*n, ray_pos);
            leaf += c;
            if (kAhead) entry = 72 + leaf;
            empty = (n->child_empty >> c) & 1u;
        }
    }
    if (empty) {
        if (kAhead && allow && empty_ahead(*ea, entry, ray_dir)) return -3;
        const float t_max = fmaxf(oct_child_exit(*n, c, ray_pos, ray_dir), 0.1f);
        ray_pos = madd3(ray_pos, ray_dir, t_max);
        return -2;
    }
    return leaf;
    }
    const OctInternal& r = oct.node[0];
    const int c1 = oct_child(r, ray_pos);
    if ((r.child_empty >> c1) & 1u) {
        if (kAhead && allow && empty_ahead(*ea, c1, ray_dir)) return -3;
        float t_max = fmaxf(oct_child_exit(r, c1, ray_pos, ray_dir), 0.1f);
        ray_pos = madd3(ray_pos, ray_dir, t_max);
        return -2;
    }
    const OctInternal& n1 = oct.node[1 + c1];
    const int c2 = oct_child(n1, ray_pos);
    if ((n1.child_empty >> c2) & 1u) {
        if (kAhead && allow && empty_ahead(*ea, 8 + c1 * 8 + c2, ray_dir)) return -3;
        float t_max = fmaxf(oct_child_exit(n1, c2, ray_pos, ray_dir), 0.1f);
        ray_pos = madd3(ray_pos, ray_dir, t_max);
        return -2;
    }
    const OctInternal& n2 = oct.node[9 + c1 * 8 + c2];
    const int c3 = oct_child(n2, ray_pos);
    if ((n2.child_empty >> c3) & 1u) {
        if (kAhead && allow && empty_ahead(*ea, 72 + c1 * 64 + c2 * 8 + c3, ray_dir)) return -3;
        float t_max = fmaxf(oct_child_exit(n2, c3, ray_pos, ray_dir), 0.1f);
        ray_pos = madd3(ray_pos, ray_dir, t_max);
        return -2;
    }
    return c1 * 64 + c2 * 8 + c3;
}

// ---- volume lookups --------------------------------------------------------------------------------
// world -> normalised texture coordinate; the operand order reproduces the reference's inlined
// `xform.transpose().inverse().transform_point(pos)` followed by `(pos - bmin) / dim`.
VPT_DEV bool volume_coord(const VolumeRec& v, float3 p, float3& uvw) {
    // mul(y), fma(x), fma(z), fma(adjugate, 1/det): the chain the reference's inlined inverse + transform_point compiles to
    float ix = pfma(v.adj3[0], v.idet, pfma(p.z, v.m[0][2], pfma(p.x, v.m[0][0], pmul(p.y, v.m[0][1]))));
    float iy = pfma(v.adj3[1], v.idet, pfma(p.z, v.m[1][2], pfma(p.x, v.m[1][0], pmul(p.y, v.m[1][1]))));
    float iz = pfma(v.adj3[2], v.idet, pfma(p.z, v.m[2][2], pfma(p.x, v.m[2][0], pmul(p.y, v.m[2][1]))));
    ix = psub(ix, v.bmin[0]); iy = psub(iy, v.bmin[1]); iz = psub(iz, v.bmin[2]);
    uvw.x = pmul(ix, v.rdim[0]); uvw.y = pmul(iy, v.rdim[1]); uvw.z = pmul(iz, v.rdim[2]);   // div.approx == rcp.approx * x
    return !(uvw.x < .0f || uvw.y < .0f || uvw.z < .0f || uvw.x > 1.0f || uvw.y > 1.0f || uvw.z > 1.0f);
}

VPT_DEV float volume_density(const VolumeRec& v, float3 p) {
    float3 uvw;
    if (!volume_coord(v, p, uvw)) return .0f;
    return tex3D<float>((cudaTextureObject_t)v.density_tex, uvw.x, uvw.y, uvw.z);
}

VPT_DEV float3 volume_color(const VolumeRec& v, float3 p) {
    if (!(v.flags & 1u)) return f3(1.0f);
    float3 uvw;
    if (!volume_coord(v, p, uvw)) return f3(.0f);
    float4 cd = tex3D<float4>((cudaTextureObject_t)v.color_tex, uvw.x, uvw.y, uvw.z);
    return f3(cd.x, cd.y, cd.z);
}

// Emission lookup: heat texture addressed with the DENSITY grid's bmin/dim (quirk Q8).
VPT_DEV float3 volume_emission(const VolumeRec& v, float3 p, const float3* lut, float pivot, float scale) {
    if (!(v.flags & 2u)) return f3(.0f);
    float3 uvw;
    if (!volume_coord(v, p, uvw)) return f3(.0f);
    float index = tex3D<float>((cudaTextureObject_t)v.emission_tex, uvw.x, uvw.y, uvw.z);
    index = clampf(index * 255.0f / pivot, .0f, 255.0f);
    return lut[int(index)] * scale;
}

// Leaf volume list: the flat CSR tables, or (level (A) entry) the caller's own OCTNode leaf.
struct LeafList { const int* idx; uint32_t n; };
VPT_DEV LeafList leaf_list_of(const SceneTables& sc, int leaf) {
    LeafList l;
    if (sc.leaf_nodes) {
        const vpt_octnode* nd = reinterpret_cast<const vpt_octnode*>(sc.leaf_nodes[leaf]);
        l.idx = nd ? nd->vol_indices : nullptr; l.n = nd ? (uint32_t)nd->num_volumes : 0u;
    } else {
        const uint2 lst = sc.leaf_list[leaf];
        l.idx = sc.leaf_indices + lst.x; l.n = lst.y;
    }
    return l;
}

VPT_DEV float leaf_density(const SceneTables& sc, const VolumeRec& vol0, int leaf, float3 p) {
    if (sc.single_volume) return 0.0f + volume_density(vol0, p);
    const LeafList lst = leaf_list_of(sc, leaf);
    float density = 0.0f;
    for (uint32_t i = 0; i < lst.n; ++i) density += volume_density(sc.volumes[lst.idx[i]], p);
    return density;
}

VPT_DEV float3 leaf_color(const SceneTables& sc, const VolumeRec& vol0, int leaf, float3 p) {
    if (sc.single_volume) return fmax3(f3(0.0f), volume_color(vol0, p));
    const LeafList lst = leaf_list_of(sc, leaf);
    float3 color = f3(0.0f);
    for (uint32_t i = 0; i < lst.n; ++i) color = fmax3(color, volume_color(sc.volumes[lst.idx[i]], p));
    return color;
}

VPT_DEV float3 leaf_emission(const SceneTables& sc, const VolumeRec& vol0, int leaf, float3 p, const float3* lut, float pivot, float scale) {
    if (sc.single_volume) return f3(0.0f) + volume_emission(vol0, p, lut, pivot, scale);
    const LeafList lst = leaf_list_of(sc, leaf);
    float3 e = f3(0.0f);
    for (uint32_t i = 0; i < lst.n; ++i) e += volume_emission(sc.volumes[lst.idx[i]], p, lut, pivot, scale);
    return e;
}

// ---- phase function ---------------------------------------------------------------------------------
VPT_DEV float hg_phase(float cos_theta, float g) {           // reference henyey_greenstein, light.h:55-64 (pi/4 scale: Q1)
    float denominator = 1 + g * g - 2 * g * cos_theta;
    return VPT_PI_4_F * (1 - g * g) / (denominator * sqrtf(denominator));
}

// returns cos_theta of the sampled deflection (the reference returns henyey_greenstein(-cos_theta, g), used by integrator 1).
// Operation order and fusion follow the reference build's SASS, not just its PTX: ptxas contracts the single-use products
// that the PTX still shows as mul + sub (1 - g*g -> fma(-g, g, 1); a*b - c*d -> fma(a, b, -(c*d)); 1 - c*c -> fma(-c, c, 1)),
// which matters when the cross products cancel (directions close to the y axis).
VPT_DEV float hg_sample(float3& wo, Rng& rng, float g) {      // reference sample_hg, render_kernel.cu:306-325
    float cos_theta;
    if (fabsf(g) < VPT_EPS) { const float u = rng.next(); cos_theta = psub(1.0f, padd(u, u)); }
    else {
        const float g2 = padd(g, g);
        const float sqr_term = pfma(-g, g, 1.0f) / pfma(g2, rng.next(), psub(1.0f, g));
        cos_theta = pfma(-sqr_term, sqr_term, pfma(g, g, 1.0f)) / g2;
    }
    const float sin_theta = sqrtf(fmaxf(pfma(-cos_theta, cos_theta, 1.0f), .0f));
    const float phi = pmul(rng.next(), (float)(2.0 * 3.14159265358979323846));
    // orthonormal frame around -wo (reference coordinate_system, :92-102)
    const float3 v1 = make_float3(-wo.x, -wo.y, -wo.z);
    float3 v2;
    if (fabsf(v1.x) > fabsf(v1.y)) v2 = f3(-v1.z, 0.0f, v1.x);
    else                           v2 = f3(0.0f, v1.z, -v1.y);
    v2 = normalize(v2);
    // cross(v1, v2) with v1 = -wo, written on wo as the compiled reference evaluates it
    float3 v3 = make_float3(pfma(wo.z, v2.y, -pmul(wo.y, v2.z)), pfma(wo.x, v2.z, -pmul(wo.z, v2.x)), pfma(wo.y, v2.x, -pmul(wo.x, v2.y)));
    v3 = normalize(v3);
    // x*sin*cos(phi) + y*sin*sin(phi) + z*cos  ->  mul(y term), fma(x term), fma(z term)
    const float cp = cosf(phi), sp = sinf(phi);
    const float3 xs = make_float3(pmul(sin_theta, v2.x), pmul(sin_theta, v2.y), pmul(sin_theta, v2.z));
    const float3 ys = make_float3(pmul(sin_theta, v3.x), pmul(sin_theta, v3.y), pmul(sin_theta, v3.z));
    wo = make_float3(pfma(wo.x, cos_theta, pfma(xs.x, cp, pmul(sp, ys.x))),
                     pfma(wo.y, cos_theta, pfma(xs.y, cp, pmul(sp, ys.y))),
                     pfma(wo.z, cos_theta, pfma(xs.z, cp, pmul(sp, ys.z))));
    return cos_theta;
}

VPT_DEV float3 sun_direction(float azimuth, float elevation) {  // reference degree_to_cartesian, :126-142
    float az = clampf(azimuth, .0f, 360.0f);
    float el = clampf(elevation, -90.0f, 90.0f);
    az = az * VPT_PI_F / 180.0f;
    el = (90.0f - el) * VPT_PI_F / 180.0f;
    float x = sinf(el) * cosf(az);
    float y = cosf(el);
    float z = sinf(el) * sinf(az);
    return normalize(f3(x, y, z));
}

} // namespace vpt
