// vpt_scene_build.cpp -- instance acceleration build behind the C ABI (SURVEY 8(f) row N1).
//
// Replaces BVH_Builder::build_bvh (source/bvh/bvh_builder.cpp:46-105): the host root set-up (:61-78), the
// depth-3 octree (bvh_kernels.cu:204-246, 582-604) and the LBVH (bvh_kernels.cu:460-580).
//   * vpt_octree_build  any number of instances.  n <= 600: a contiguous 585-node tree in the reference's OCTNode
//                       layout (either kernel can consume it).  n > 600 (the reference overflows vol_indices[600],
//                       quirk Q11): only the root record exists in that layout; the octree itself lives in the flat
//                       tables (73 internal nodes + 512 CSR leaf lists) that are built for EVERY n and registered
//                       under the root pointer -- this library's render path reads those.
//   * vpt_bvh_build     Karras LBVH in the reference's BVHNode layout (node arrays + sorted Morton codes / ids).
#include "vpt_host.h"

#include <cstdlib>
#include <cstring>
#include <cmath>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

namespace vpt {

static std::mutex g_reg_mutex;
static std::unordered_map<vpt_devptr_t, SceneEntry> g_registry;
static unsigned long long g_generation = 0;

bool scene_registry_find(vpt_devptr_t d_root, SceneEntry* out) {
    std::lock_guard<std::mutex> lk(g_reg_mutex);
    auto it = g_registry.find(d_root);
    if (it == g_registry.end()) return false;
    if (out) *out = it->second;
    return true;
}

static void free_entry(SceneEntry& e) {
    cudaFree(e.d_internal); cudaFree(e.d_leaf_list); cudaFree(e.d_leaf_indices);
    e.d_internal = nullptr; e.d_leaf_list = nullptr; e.d_leaf_indices = nullptr;
}

// the three halvings of divide_bbox (bvh_kernels.cu:150-202) on the host: float sum, times 0.5 (exact)
static void child_box_host(int idx, const float pmin[3], const float pmax[3], float cmin[3], float cmax[3]) {
    const float hx = (float)((double)(pmin[0] + pmax[0]) * 0.5), hy = (float)((double)(pmin[1] + pmax[1]) * 0.5), hz = (float)((double)(pmin[2] + pmax[2]) * 0.5);
    const bool xp = idx & 1, ym = idx & 2, zp = idx & 4;
    cmin[0] = xp ? hx : pmin[0]; cmin[1] = ym ? pmin[1] : hy; cmin[2] = zp ? hz : pmin[2];
    cmax[0] = xp ? pmax[0] : hx; cmax[1] = ym ? hy : pmax[1]; cmax[2] = zp ? pmax[2] : hz;
}

} // namespace vpt

using vpt::fail_global;

extern "C" {

void vpt_volume_bounds(const vpt_gpu_vdb* v, float out6[6]) { vpt::instance_bounds_host(*v, out6); }

int vpt_octree_build(const vpt_gpu_vdb* h_volumes, int n, vpt_devptr_t* d_root_out) {
    if (!h_volumes || !d_root_out || n < 1) return fail_global(VPT_ERR_INVALID, "vpt_octree_build: bad arguments");
    *d_root_out = 0;
    int device = 0;
    if (cudaGetDevice(&device) != cudaSuccess) return fail_global(VPT_ERR_CUDA, "vpt_octree_build: no CUDA device");

    // root exactly as the reference host code builds it (union of instance bounds, +-1 world unit), bvh_builder.cpp:61-78
    vpt_octnode* root = (vpt_octnode*)calloc(1, sizeof(vpt_octnode));
    if (!root) return fail_global(VPT_ERR_IO, "vpt_octree_build: out of memory");
    root->bbox.pmin = { 3.402823466e+38F, 3.402823466e+38F, 3.402823466e+38F };
    root->bbox.pmax = { -3.402823466e+38F, -3.402823466e+38F, -3.402823466e+38F };
    root->max_extinction = .0f; root->min_extinction = 3.402823466e+38F; root->voxel_size = 3.402823466e+38F;
    root->depth = 4;
    unsigned any_flags = 0;
    unsigned long long max_grid_bytes = 0;
    for (int i = 0; i < n; ++i) {
        const vpt_i3 dm = h_volumes[i].vdb_info.dim;
        const unsigned long long gb = (dm.x > 0 && dm.y > 0 && dm.z > 0) ? 4ull * (unsigned long long)dm.x * (unsigned long long)dm.y * (unsigned long long)dm.z : 0ull;
        if (gb > max_grid_bytes) max_grid_bytes = gb;
        float b[6]; vpt::instance_bounds_host(h_volumes[i], b);
        root->bbox.pmax.x = fmaxf(root->bbox.pmax.x, b[3]); root->bbox.pmax.y = fmaxf(root->bbox.pmax.y, b[4]); root->bbox.pmax.z = fmaxf(root->bbox.pmax.z, b[5]);
        root->bbox.pmin.x = fminf(root->bbox.pmin.x, b[0]); root->bbox.pmin.y = fminf(root->bbox.pmin.y, b[1]); root->bbox.pmin.z = fminf(root->bbox.pmin.z, b[2]);
        if (i < VPT_OCT_MAX_VOLUMES) root->vol_indices[i] = i;          // the reference writes past the array here (Q11)
        root->num_volumes++;
        root->max_extinction = fmaxf(root->max_extinction, h_volumes[i].vdb_info.max_density);
        root->min_extinction = fminf(root->min_extinction, h_volumes[i].vdb_info.min_density);
        root->has_children = 1;
        any_flags |= (h_volumes[i].vdb_info.has_color ? 1u : 0u) | (h_volumes[i].vdb_info.has_emission ? 2u : 0u);
    }
    root->bbox.pmax.x += 1.0f; root->bbox.pmax.y += 1.0f; root->bbox.pmax.z += 1.0f;
    root->bbox.pmin.x -= 1.0f; root->bbox.pmin.y -= 1.0f; root->bbox.pmin.z -= 1.0f;

    const bool ref_layout = n <= VPT_OCT_MAX_VOLUMES;
    const size_t node_count = ref_layout ? 585 : 1;
    vpt_octnode* d_nodes = nullptr; vpt_gpu_vdb* d_vols = nullptr; void* d_bounds = nullptr;
    vpt::SceneEntry ent; ent.device = device; ent.n = n;
    ent.root6[0] = root->bbox.pmin.x; ent.root6[1] = root->bbox.pmin.y; ent.root6[2] = root->bbox.pmin.z;
    ent.root6[3] = root->bbox.pmax.x; ent.root6[4] = root->bbox.pmax.y; ent.root6[5] = root->bbox.pmax.z;
    ent.max_extinction = root->max_extinction; ent.min_extinction = root->min_extinction; ent.any_flags = any_flags; ent.max_grid_bytes = max_grid_bytes;
    ent.dim0[0] = h_volumes[0].vdb_info.dim.x; ent.dim0[1] = h_volumes[0].vdb_info.dim.y; ent.dim0[2] = h_volumes[0].vdb_info.dim.z;
    std::vector<int> counts(585);
    std::vector<vpt::OctInternal> internal(vpt::kOctInternalNodes);
    std::vector<uint2> leaf_list(vpt::kOctLeaves);

    cudaError_t e = cudaMalloc(&d_nodes, sizeof(vpt_octnode) * node_count);
    if (e == cudaSuccess) e = cudaMemset(d_nodes, 0, sizeof(vpt_octnode) * node_count);
    if (e == cudaSuccess) e = cudaMemcpy(d_nodes, root, sizeof(vpt_octnode), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMalloc(&d_vols, sizeof(vpt_gpu_vdb) * (size_t)n);
    if (e == cudaSuccess) e = cudaMemcpy(d_vols, h_volumes, sizeof(vpt_gpu_vdb) * (size_t)n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && ref_layout) e = vpt::octree_build_device(d_nodes, d_vols, n, 0);
    free(root);

    // flat tables: per-node instance counts -> internal records + CSR offsets on the host -> leaf lists on the device
    if (e == cudaSuccess) e = vpt::octree_flat_counts(d_vols, n, ent.root6, &d_bounds, counts.data(), 0);
    if (e == cudaSuccess) {
        // boxes of the internal nodes, by the reference's halving arithmetic
        std::vector<float> bmin(73 * 3), bmax(73 * 3);
        for (int a = 0; a < 3; ++a) { bmin[a] = ent.root6[a]; bmax[a] = ent.root6[3 + a]; }
        for (int j = 1; j < 73; ++j) {
            const int parent = j < 9 ? 0 : 1 + ((j - 9) >> 3), c = j < 9 ? j - 1 : (j - 9) & 7;
            vpt::child_box_host(c, &bmin[parent * 3], &bmax[parent * 3], &bmin[j * 3], &bmax[j * 3]);
        }
        for (int j = 0; j < 73; ++j) {
            vpt::OctInternal o; memset(&o, 0, sizeof(o)); o.child_empty = 0xffu;
            const bool parent_ok = j == 0 || counts[j < 9 ? 0 : 1 + ((j - 9) >> 3)] > 0;
            if (parent_ok && counts[j] > 0) {
                float c0min[3], c0max[3];
                vpt::child_box_host(0, &bmin[j * 3], &bmax[j * 3], c0min, c0max);      // child 0 = (x-, y+, z-)
                for (int a = 0; a < 3; ++a) { o.pmin[a] = bmin[j * 3 + a]; o.pmax[a] = bmax[j * 3 + a]; }
                o.half[0] = c0max[0]; o.half[1] = c0min[1]; o.half[2] = c0max[2];
                const int first = j == 0 ? 1 : j < 9 ? 9 + (j - 1) * 8 : 73 + (j - 9) * 8;
                uint32_t mask = 0;
                for (int c = 0; c < 8; ++c) if (counts[first + c] == 0) mask |= 1u << c;
                o.child_empty = mask;
            }
            internal[j] = o;
        }
        size_t total = 0;
        for (int l = 0; l < 512; ++l) {
            // a leaf exists only under populated ancestors; overlap with a child implies overlap with its parent, so count > 0 suffices
            leaf_list[l] = make_uint2((unsigned)total, (unsigned)counts[73 + l]);
            total += (size_t)counts[73 + l];
            if (counts[73 + l] > ent.max_leaf_count) ent.max_leaf_count = counts[73 + l];
        }
        ent.total_indices = total;
        e = cudaMalloc(&ent.d_internal, sizeof(vpt::OctInternal) * vpt::kOctInternalNodes);
        if (e == cudaSuccess) e = cudaMalloc(&ent.d_leaf_list, sizeof(uint2) * vpt::kOctLeaves);
        if (e == cudaSuccess) e = cudaMalloc(&ent.d_leaf_indices, sizeof(int) * (total ? total : 1));
        if (e == cudaSuccess) e = cudaMemcpy(ent.d_internal, internal.data(), sizeof(vpt::OctInternal) * vpt::kOctInternalNodes, cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMemcpy(ent.d_leaf_list, leaf_list.data(), sizeof(uint2) * vpt::kOctLeaves, cudaMemcpyHostToDevice);
        if (e == cudaSuccess && total) {
            // offsets are the .x members of the (offset, count) pairs: hand the kernel a packed copy
            std::vector<unsigned> offs(512); for (int l = 0; l < 512; ++l) offs[l] = leaf_list[l].x;
            unsigned* d_offs = nullptr;
            e = cudaMalloc(&d_offs, sizeof(unsigned) * 512);
            if (e == cudaSuccess) e = cudaMemcpy(d_offs, offs.data(), sizeof(unsigned) * 512, cudaMemcpyHostToDevice);
            if (e == cudaSuccess) e = vpt::octree_flat_fill(d_bounds, n, ent.root6, d_offs, ent.d_leaf_indices, 0);
            if (e == cudaSuccess) e = cudaDeviceSynchronize();
            cudaFree(d_offs);
        }
    }
    cudaFree(d_bounds);
    cudaFree(d_vols);
    if (e != cudaSuccess) {
        cudaFree(d_nodes); vpt::free_entry(ent);
        return fail_global(VPT_ERR_CUDA, std::string("vpt_octree_build: ") + cudaGetErrorString(e));
    }
    {
        std::lock_guard<std::mutex> lk(vpt::g_reg_mutex);
        ent.generation = ++vpt::g_generation;
        vpt::g_registry[(vpt_devptr_t)(uintptr_t)d_nodes] = ent;
    }
    *d_root_out = (vpt_devptr_t)(uintptr_t)d_nodes;
    return VPT_OK;
}

int vpt_octree_info(vpt_devptr_t d_root, int* n_instances, int* reference_layout, long long* total_leaf_entries, int* max_leaf_entries) {
    vpt::SceneEntry e;
    if (!vpt::scene_registry_find(d_root, &e)) return fail_global(VPT_ERR_INVALID, "vpt_octree_info: not an octree built by vpt_octree_build");
    if (n_instances) *n_instances = e.n;
    if (reference_layout) *reference_layout = e.n <= VPT_OCT_MAX_VOLUMES ? 1 : 0;
    if (total_leaf_entries) *total_leaf_entries = (long long)e.total_indices;
    if (max_leaf_entries) *max_leaf_entries = e.max_leaf_count;
    return VPT_OK;
}

int vpt_octree_read(vpt_devptr_t d_root, vpt_octnode* h_nodes585, int* h_exists585) {
    if (!d_root || !h_nodes585 || !h_exists585) return fail_global(VPT_ERR_INVALID, "vpt_octree_read: null argument");
    vpt::SceneEntry ent;
    if (vpt::scene_registry_find(d_root, &ent) && ent.n > VPT_OCT_MAX_VOLUMES)
        return fail_global(VPT_ERR_UNSUPPORTED, "vpt_octree_read: an octree over more than 600 instances has no reference-layout nodes (use vpt_octree_read_flat)");
    cudaError_t e = vpt::octree_snapshot(reinterpret_cast<const vpt_octnode*>((uintptr_t)d_root), h_nodes585, h_exists585);
    if (e != cudaSuccess) return fail_global(VPT_ERR_CUDA, std::string("vpt_octree_read: ") + cudaGetErrorString(e));
    return VPT_OK;
}

int vpt_octree_read_flat(vpt_devptr_t d_root, unsigned leaf_offset_count[1024], int* indices, long long capacity) {
    vpt::SceneEntry ent;
    if (!leaf_offset_count || !vpt::scene_registry_find(d_root, &ent)) return fail_global(VPT_ERR_INVALID, "vpt_octree_read_flat: not an octree built by vpt_octree_build");
    cudaError_t e = cudaMemcpy(leaf_offset_count, ent.d_leaf_list, sizeof(uint2) * 512, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && indices) {
        if (capacity < (long long)ent.total_indices) return fail_global(VPT_ERR_INVALID, "vpt_octree_read_flat: index buffer too small");
        if (ent.total_indices) e = cudaMemcpy(indices, ent.d_leaf_indices, sizeof(int) * ent.total_indices, cudaMemcpyDeviceToHost);
    }
    if (e != cudaSuccess) return fail_global(VPT_ERR_CUDA, std::string("vpt_octree_read_flat: ") + cudaGetErrorString(e));
    return VPT_OK;
}

int vpt_octree_destroy(vpt_devptr_t d_root) {
    if (!d_root) return VPT_OK;
    vpt::SceneEntry ent; bool found = false;
    {
        std::lock_guard<std::mutex> lk(vpt::g_reg_mutex);
        auto it = vpt::g_registry.find(d_root);
        if (it != vpt::g_registry.end()) { ent = it->second; vpt::g_registry.erase(it); found = true; }
    }
    if (found) vpt::free_entry(ent);
    cudaFree((void*)(uintptr_t)d_root);
    return VPT_OK;
}

int vpt_bvh_build(const vpt_gpu_vdb* h_volumes, int n, vpt_devptr_t* d_nodes_out, vpt_devptr_t* d_leaves_out, float scene_bounds6[6],
                  unsigned long long* h_sorted_codes, int* h_sorted_ids) {
    if (!h_volumes || n < 1 || !d_nodes_out || !d_leaves_out) return fail_global(VPT_ERR_INVALID, "vpt_bvh_build: bad arguments");
    *d_nodes_out = 0; *d_leaves_out = 0;
    vpt_gpu_vdb* d_vols = nullptr; vpt_bvhnode *d_nodes = nullptr, *d_leaves = nullptr;
    const size_t n_int = n > 1 ? (size_t)n - 1 : 1;
    cudaError_t e = cudaMalloc(&d_vols, sizeof(vpt_gpu_vdb) * (size_t)n);
    if (e == cudaSuccess) e = cudaMemcpy(d_vols, h_volumes, sizeof(vpt_gpu_vdb) * (size_t)n, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMalloc(&d_nodes, sizeof(vpt_bvhnode) * n_int);
    if (e == cudaSuccess) e = cudaMalloc(&d_leaves, sizeof(vpt_bvhnode) * (size_t)n);
    if (e == cudaSuccess) e = cudaMemset(d_nodes, 0, sizeof(vpt_bvhnode) * n_int);
    if (e == cudaSuccess) e = cudaMemset(d_leaves, 0, sizeof(vpt_bvhnode) * (size_t)n);
    if (e == cudaSuccess) e = vpt::bvh_build_device(d_vols, n, d_nodes, d_leaves, scene_bounds6, h_sorted_codes, h_sorted_ids, 0);
    cudaFree(d_vols);
    if (e != cudaSuccess) { cudaFree(d_nodes); cudaFree(d_leaves); return fail_global(VPT_ERR_CUDA, std::string("vpt_bvh_build: ") + cudaGetErrorString(e)); }
    *d_nodes_out = (vpt_devptr_t)(uintptr_t)d_nodes; *d_leaves_out = (vpt_devptr_t)(uintptr_t)d_leaves;
    return VPT_OK;
}

// Copies a BVH in the reference layout (this builder's or the reference's) to the host with its pointers turned into
// indices: internal node i -> i, leaf i -> (n - 1) + i, null / outside both arrays -> -1 (stored in the pointer fields).
int vpt_bvh_read(vpt_devptr_t d_nodes, vpt_devptr_t d_leaves, int n, vpt_bvhnode* h_nodes, vpt_bvhnode* h_leaves) {
    if (!d_leaves || n < 1 || !h_leaves || (n > 1 && (!d_nodes || !h_nodes))) return fail_global(VPT_ERR_INVALID, "vpt_bvh_read: bad arguments");
    cudaError_t e = cudaMemcpy(h_leaves, (const void*)(uintptr_t)d_leaves, sizeof(vpt_bvhnode) * (size_t)n, cudaMemcpyDeviceToHost);
    if (e == cudaSuccess && n > 1) e = cudaMemcpy(h_nodes, (const void*)(uintptr_t)d_nodes, sizeof(vpt_bvhnode) * (size_t)(n - 1), cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) return fail_global(VPT_ERR_CUDA, std::string("vpt_bvh_read: ") + cudaGetErrorString(e));
    auto to_index = [&](vpt_devptr_t p) -> vpt_devptr_t {
        const uint64_t nb = d_nodes, lb = d_leaves, sz = sizeof(vpt_bvhnode);
        if (n > 1 && p >= nb && p < nb + sz * (uint64_t)(n - 1) && (p - nb) % sz == 0) return (p - nb) / sz;
        if (p >= lb && p < lb + sz * (uint64_t)n && (p - lb) % sz == 0) return (uint64_t)(n - 1) + (p - lb) / sz;
        return (vpt_devptr_t)(int64_t)-1;
    };
    for (int i = 0; i < n; ++i) { h_leaves[i].leftChild = to_index(h_leaves[i].leftChild); h_leaves[i].rightChild = to_index(h_leaves[i].rightChild); h_leaves[i].parent = to_index(h_leaves[i].parent); }
    for (int i = 0; i + 1 < n; ++i) { h_nodes[i].leftChild = to_index(h_nodes[i].leftChild); h_nodes[i].rightChild = to_index(h_nodes[i].rightChild); h_nodes[i].parent = to_index(h_nodes[i].parent); }
    return VPT_OK;
}

int vpt_bvh_destroy(vpt_devptr_t d_nodes, vpt_devptr_t d_leaves) {
    if (d_nodes) cudaFree((void*)(uintptr_t)d_nodes);
    if (d_leaves) cudaFree((void*)(uintptr_t)d_leaves);
    return VPT_OK;
}

} // extern "C"
