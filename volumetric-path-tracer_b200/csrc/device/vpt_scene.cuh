// vpt_scene.cuh -- the flattened, HBM-resident scene tables the wavefront kernels read.
//
// The reference walks 2520-byte pointer-linked OCTNodes from the device heap and re-inverts each
// volume's 4x4 transform at every density lookup (render_kernel.cu:984-1001, :1102-1115).  Here a
// one-off prepare kernel turns the very same inputs (GPU_VDB[] + OCTNode tree, i.e. the launch
// parameters of the reference kernel) into:
//   * OctInternal[73]   : root + 8 + 64 internal nodes, 48 B each (pmin/half/pmax + child-empty mask)
//                         -> staged into shared memory by every CTA (3.5 KB);
//   * leaf volume lists : 512 (offset,count) pairs + a flat index array (instanced scenes only);
//   * VolumeRec[N]      : world->texture affine as the reference's own adjugate/determinant split,
//                         so the lookup coordinate is bit-identical to the reference's inline inverse.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <cuda_runtime.h>

namespace vpt {

constexpr int kOctInternalNodes = 73;     // 1 + 8 + 64
constexpr int kOctLeaves        = 512;

struct __align__(16) OctInternal {        // 48 B
    float pmin[3];
    float half[3];                        // split planes = children[0].pmax.x / .pmin.y / .pmax.z
    float pmax[3];
    uint32_t child_empty;                 // bit c set: child c has num_volumes == 0 (skip it)
    uint32_t pad[2];
};

struct __align__(16) VolumeRec {          // 96 B
    float m[3][3];        // m[r][c] = round(adj[c][r] * idet): coefficient of world (x,y,z)[c] for index coord r
    float adj3[3];        // unscaled adjugate translation term of row r (fused with idet at lookup time)
    float idet;           // rcp.approx(det)
    float bmin[3];        // vdb_info.bmin
    float rdim[3];        // rcp.approx(float(dim))  (div.approx == MUFU.RCP + FMUL)
    uint32_t flags;       // bit0 has_color, bit1 has_emission
    unsigned long long density_tex, emission_tex, color_tex;
};

struct SceneTables {
    float root_pmin[3], root_pmax[3];
    float max_extinction, min_extinction;   // root values: the only majorant/minorant the live code uses
    int   num_volumes;
    int   single_volume;                    // 1: every non-empty leaf lists exactly volume 0
    const OctInternal* internal;            // [73]
    const uint2*       leaf_list;           // [512] (offset, count) into leaf_indices
    const int*         leaf_indices;
    const VolumeRec*   volumes;             // [num_volumes]
    // level (A) entry only (vpt_level_a.cu): leaves read straight from the caller's pointer-linked OCTNodes, no flat lists.
    // Null everywhere else.  [512] pointers to the leaf nodes (null where the leaf does not exist).
    const void* const* leaf_nodes;
};

// "Nothing populated ahead" (DESIGN.md section 8j, build_empty_ahead in vpt_walk.cuh): one entry per (node, child) pair below the root,
// entry of child c of internal node i at i * 8 + c.  Bit o of an entry: no populated leaf in the orthant of the entry's block for octant o.
constexpr int kAheadEntries = 8 + 64 + 512;
struct __align__(16) EmptyAhead { uint8_t bit[kAheadEntries + 8]; };

// The context's scene allocation: the tables, then the empty-ahead table of the current render call.  k_empty_ahead writes the table
// once per call; k_generate and the lean k_trace stage it into shared memory with the octree (load_frame_shared), reaching it through
// FrameArgs::scene, so no kernel's parameter block changes.
struct SceneAlloc { SceneTables sc; EmptyAhead ahead; };
static_assert(sizeof(EmptyAhead) % 16 == 0 && offsetof(SceneAlloc, ahead) % 16 == 0, "the table is staged in 16-byte words");

} // namespace vpt
