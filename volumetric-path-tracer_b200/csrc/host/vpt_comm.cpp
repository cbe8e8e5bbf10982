// vpt_comm.cpp -- the multi-GPU exchange step of the path, issued from the C++ host (SURVEY 8(e)).
//
// One process per GPU.  The frame is sharded by interleaved row stripes (vpt_set_partition), the scene is replicated, and
// pixels are independent (every Philox stream is keyed by the GLOBAL pixel index), so a pass needs no data-path collective.
// The only exchange is the gather of the rank-local frames: one ncclAllGather of the accumulators (and optionally of the
// packed display words) per vpt_render_pass(es) call, followed by k_unpermute into the caller's full-frame buffer.  It is
// enqueued by vpt_render_passes itself, right behind the last resolve kernel:
//   * default: on the caller's stream (in order, nothing else to synchronise);
//   * option "gather_async" = 1: on the context's side stream behind an event, so that the NEXT call's generate / trace
//     kernels overlap it; the library makes the next call wait only where it would overwrite the accumulator, and
//     vpt_comm_wait() joins the side stream into the caller's stream.
//
// NCCL is bound at run time (dlopen of the copy the process already uses -- torch.distributed's -- else libnccl.so.2), so the
// library loads and renders on hosts without NCCL; only vpt_comm_* needs it.  The reference has no multi-GPU path: there
// is nothing to be compatible with here except "the gathered frame equals the single-GPU frame bit for bit" (tested).
#include "vpt_host.h"

#include <dlfcn.h>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>

namespace {

typedef struct { char internal[128]; } nccl_unique_id;      // ncclUniqueId (nccl.h:37-38)
typedef void* nccl_comm_t;
typedef int nccl_result_t;                                    // ncclSuccess == 0
enum { NCCL_CHAR = 0, NCCL_FLOAT32 = 7 };                     // ncclDataType_t values (nccl.h)

struct NcclApi {
    void* handle = nullptr;
    nccl_result_t (*GetUniqueId)(nccl_unique_id*) = nullptr;
    nccl_result_t (*CommInitRank)(nccl_comm_t*, int, nccl_unique_id, int) = nullptr;
    nccl_result_t (*CommDestroy)(nccl_comm_t) = nullptr;
    nccl_result_t (*AllGather)(const void*, void*, size_t, int, nccl_comm_t, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(nccl_result_t) = nullptr;
    nccl_result_t (*GetVersion)(int*) = nullptr;
    std::string error;
};

NcclApi& nccl() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        const char* names[] = { "libnccl.so.2", "libnccl.so" };
        for (const char* n : names) { api.handle = dlopen(n, RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL); if (api.handle) break; }   // the copy already in the process
        for (const char* n : names) { if (api.handle) break; api.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL); }
        if (!api.handle) { api.error = std::string("NCCL not found (dlopen libnccl.so.2): ") + (dlerror() ? dlerror() : "?"); return; }
        auto sym = [&](const char* s) { void* p = dlsym(api.handle, s); if (!p && api.error.empty()) api.error = std::string("NCCL symbol missing: ") + s; return p; };
        api.GetUniqueId = (decltype(api.GetUniqueId))sym("ncclGetUniqueId");
        api.CommInitRank = (decltype(api.CommInitRank))sym("ncclCommInitRank");
        api.CommDestroy = (decltype(api.CommDestroy))sym("ncclCommDestroy");
        api.AllGather = (decltype(api.AllGather))sym("ncclAllGather");
        api.GetErrorString = (decltype(api.GetErrorString))sym("ncclGetErrorString");
        api.GetVersion = (decltype(api.GetVersion))sym("ncclGetVersion");
    });
    return api;
}

int nccl_fail(vpt_context* c, const char* what, nccl_result_t r) {
    NcclApi& n = nccl();
    return vpt::fail_ctx(c, VPT_ERR_CUDA, std::string(what) + ": NCCL error " + std::to_string(r) + " (" + (n.GetErrorString ? n.GetErrorString(r) : "?") + ")");
}

} // namespace

#define VPT_CU(c, call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) \
    return vpt::fail_ctx(c, VPT_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); } while (0)

namespace vpt {

int comm_before_accum_write(vpt_context* c, cudaStream_t stream) {
    if (c->gather_pending) { VPT_CU(c, cudaStreamWaitEvent(stream, c->ev_gather_done, 0)); c->gather_pending = false; }
    return VPT_OK;
}

int comm_gather_frame(vpt_context* c, const FrameGeom& g, const void* d_local_accum, const void* d_local_display, cudaStream_t stream) {
    NcclApi& n = nccl();
    cudaStream_t s = stream;
    if (c->gather_async) {
        VPT_CU(c, cudaEventRecord(c->ev_render_done, stream));
        VPT_CU(c, cudaStreamWaitEvent(c->comm_stream, c->ev_render_done, 0));
        s = c->comm_stream;
    }
    const size_t px = (size_t)g.n_local;
    if (c->d_full_accum) {
        const size_t need = px * 12 * (size_t)g.n_ranks;
        if (need > c->cap_gathered) { cudaFree(c->d_gathered); c->d_gathered = nullptr; c->cap_gathered = 0; VPT_CU(c, cudaMalloc(&c->d_gathered, need)); c->cap_gathered = need; }
        nccl_result_t r = n.AllGather(d_local_accum, c->d_gathered, px * 3, NCCL_FLOAT32, (nccl_comm_t)c->nccl_comm, s);
        if (r != 0) return nccl_fail(c, "ncclAllGather(accum)", r);
        VPT_CU(c, launch_unpermute(c->d_gathered, c->d_full_accum, g, 12, s));
        c->launches++;
    }
    if (c->d_full_display) {
        const size_t need = px * 4 * (size_t)g.n_ranks;
        if (need > c->cap_gathered_disp) { cudaFree(c->d_gathered_disp); c->d_gathered_disp = nullptr; c->cap_gathered_disp = 0; VPT_CU(c, cudaMalloc(&c->d_gathered_disp, need)); c->cap_gathered_disp = need; }
        nccl_result_t r = n.AllGather(d_local_display, c->d_gathered_disp, px * 4, NCCL_CHAR, (nccl_comm_t)c->nccl_comm, s);
        if (r != 0) return nccl_fail(c, "ncclAllGather(display)", r);
        VPT_CU(c, launch_unpermute(c->d_gathered_disp, c->d_full_display, g, 4, s));
        c->launches++;
    }
    if (c->gather_async) { VPT_CU(c, cudaEventRecord(c->ev_gather_done, s)); c->gather_pending = true; }
    return VPT_OK;
}

// ---- peer-memory exchange ---------------------------------------------------------------------------------------------------------
// Block layout: header (u64 flag arrays: ready[16] done[16] error[1], adapt[16] at kPeerFlagsAdapt) | float3 accum [H][W] | u32 display
// [H][W] (exported with display only) | u32 pass counts [H][W] | f32 relative errors [H][W] | u32 active-tile count per rank [16].
// The last three serve vpt_render_adaptive.  Then, in VPT_LAYER_* bit order, one [H][W] plane of each exported layer (f32 depth and alpha,
// float3 the others), the motion vectors [H][W] float3 (VPT_LAYER_MOTION), then the binned layers: deep slices [n_slices][H][W] float4 and
// mattes [n_mattes][H][W] float4.  Each part starts on a 256-byte boundary.  Sizes and offsets are size_t: K x H x W x 16 passes 32 bits at modest frames.
static constexpr size_t kP2pHeader = 512;
static size_t p2p_round(size_t b) { return (b + 255) & ~(size_t)255; }
static size_t p2p_accum_bytes(size_t px) { return p2p_round(px * 12); }
static size_t p2p_plane_bytes(size_t px) { return p2p_round(px * 4); }
static size_t p2p_tiles_offset(size_t px, bool display) { return kP2pHeader + p2p_accum_bytes(px) + (display ? p2p_plane_bytes(px) : 0) + 2 * p2p_plane_bytes(px); }
enum BinnedLayer : int { BL_DEEP = 0, BL_MATTES = 1, kBinnedLayers = 2 };
// The motion-vector plane is not one of k_layers_publish's ExchangeLayer slots (its parameter block stays as it is): its bit lies past them,
// bit 7 stays unknown, and comm_p2p_layers publishes it with a launch of its own.
static constexpr unsigned kMotionLayerBit = VPT_LAYER_MOTION;
static_assert(kMotionLayerBit > (1u << kExchangeLayers), "the motion bit lies past the k_layers_publish layers");
// the block of a w x h frame; layer_off[l] (may be null) = byte offset of layer l's plane, 0 for a layer not in `layers`; bin_off[b] (may
// be null) = byte offset of the deep-slice (BL_DEEP) and matte (BL_MATTES) arrays, 0 for a count of 0; motion_off (may be null) = byte
// offset of the motion-vector plane, 0 without VPT_LAYER_MOTION
static size_t p2p_block_layout(size_t w, size_t h, bool display, unsigned layers, unsigned n_slices, unsigned n_mattes,
                               size_t layer_off[kExchangeLayers], size_t bin_off[kBinnedLayers] = nullptr, size_t* motion_off = nullptr)
{
    const size_t px = w * h;
    size_t end = p2p_tiles_offset(px, display) + sizeof(unsigned) * kPeerFlagStride;
    if (layers || n_slices || n_mattes) end = p2p_round(end);
    for (int l = 0; l < kExchangeLayers; ++l) {
        const bool on = (layers >> l) & 1u;
        if (layer_off) layer_off[l] = on ? end : 0;
        if (on) end += p2p_round(px * (l < XL_VOLUME ? 4 : 12));
    }
    if (motion_off) *motion_off = (layers & kMotionLayerBit) ? end : 0;
    if (layers & kMotionLayerBit) end += p2p_round(px * 12);
    const unsigned bins[kBinnedLayers] = {n_slices, n_mattes};
    for (int b = 0; b < kBinnedLayers; ++b) {
        if (bin_off) bin_off[b] = bins[b] ? end : 0;
        end += p2p_round(px * bins[b] * sizeof(float4));
    }
    return end;
}
static size_t p2p_accum_bytes(const vpt_context* c) { return p2p_accum_bytes((size_t)c->p2p_w * c->p2p_h); }
static size_t p2p_plane_bytes(const vpt_context* c) { return p2p_plane_bytes((size_t)c->p2p_w * c->p2p_h); }
static size_t p2p_count_offset(const vpt_context* c) { return kP2pHeader + p2p_accum_bytes(c) + (c->p2p_display ? p2p_plane_bytes(c) : 0); }
static size_t p2p_err_offset(const vpt_context* c) { return p2p_count_offset(c) + p2p_plane_bytes(c); }
static size_t p2p_tiles_offset(const vpt_context* c) { return p2p_tiles_offset((size_t)c->p2p_w * c->p2p_h, c->p2p_display); }
static unsigned long long* p2p_flags(void* block) { return reinterpret_cast<unsigned long long*>(block); }
static constexpr unsigned kPublishedLayers = (1u << kExchangeLayers) - 1;     // the layers k_layers_publish carries
static constexpr unsigned kLayerMask = kPublishedLayers | kMotionLayerBit;
// Header slot after the error word: what the block was exported for -- width (bits 0-27), height (28-55), display (56), layers (57-63).
// Every rank's must equal every other's: a rank exported with more planes would store past the end of its peers' blocks.  28 bits hold
// any size a partitioned frame can have (at most 65535 per side).
static constexpr int kP2pLayoutSlot = 2 * kPeerFlagStride + 1;
static unsigned long long p2p_layout_word(const vpt_context* c)
{
    return ((unsigned long long)c->p2p_w & 0xfffffffull) | (((unsigned long long)c->p2p_h & 0xfffffffull) << 28) |
           ((unsigned long long)(c->p2p_display ? 1 : 0) << 56) | ((unsigned long long)(c->p2p_layers & kPublishedLayers) << 57);
}
static std::string hex2(unsigned v) { char b[16]; snprintf(b, sizeof b, "0x%02x", v); return b; }
static std::string p2p_layout_text(unsigned long long w)
{
    return std::to_string(w & 0xfffffffull) + " x " + std::to_string((w >> 28) & 0xfffffffull) + ", display " + std::to_string((w >> 56) & 1ull) +
           ", layers " + hex2((unsigned)(w >> 57));
}
// The header slot after the layout word: the binned layers' counts -- deep slices (bits 0-31) and mattes (32-63).  The layout word is full,
// and the counts must agree for the same reason: a rank exported with more slices would store past the end of its peers' blocks.
static constexpr int kP2pBinnedSlot = kP2pLayoutSlot + 1;
static_assert(kP2pBinnedSlot < 3 * kPeerFlagStride, "the binned counts live in an unused slot of the header, before the adapt flags");
static unsigned long long p2p_binned_word(const vpt_context* c) { return (unsigned long long)c->p2p_slices | ((unsigned long long)c->p2p_mattes << 32); }
// The slot after the binned counts: the whole layer mask, whose motion bit the layout word has no room for
static constexpr int kP2pLayersSlot = kP2pBinnedSlot + 1;
static_assert(kP2pLayersSlot < 3 * kPeerFlagStride, "the layer mask lives in an unused slot of the header, before the adapt flags");
static std::string p2p_binned_text(unsigned long long w)
{
    return std::to_string(w & 0xffffffffull) + " deep slices and " + std::to_string(w >> 32) + " mattes";
}
// every mapped peer block must carry this rank's layout word and binned counts
static int p2p_check_layouts(vpt_context* c, const char* fn)
{
    const unsigned long long mine = p2p_layout_word(c), mine_bins = p2p_binned_word(c);
    for (int p = 0; p < c->p2p_n; ++p) {
        if (p == c->rank) continue;
        unsigned long long w[3] = {0, 0, 0};
        VPT_CU(c, cudaMemcpy(w, p2p_flags(c->p2p_peer[p]) + kP2pLayoutSlot, sizeof(w), cudaMemcpyDefault));
        if (w[0] != mine)
            return fail_ctx(c, VPT_ERR_INVALID, std::string(fn) + ": rank " + std::to_string(p) + " exported its block for " + p2p_layout_text(w[0]) +
                                                ", this rank (" + std::to_string(c->rank) + ") for " + p2p_layout_text(mine) +
                                                "; every rank must export the same frame size, display and layers");
        if (w[1] != mine_bins)
            return fail_ctx(c, VPT_ERR_INVALID, std::string(fn) + ": rank " + std::to_string(p) + " exported its block with " + p2p_binned_text(w[1]) +
                                                ", this rank (" + std::to_string(c->rank) + ") with " + p2p_binned_text(mine_bins) +
                                                "; every rank must export the same deep-slice and matte counts (vpt_comm_p2p_export_binned)");
        if (w[2] != c->p2p_layers)
            return fail_ctx(c, VPT_ERR_INVALID, std::string(fn) + ": rank " + std::to_string(p) + " exported its block with layers " +
                                                hex2((unsigned)w[2]) + ", this rank (" + std::to_string(c->rank) + ") with " + hex2(c->p2p_layers) +
                                                "; every rank must export the same layers");
    }
    return VPT_OK;
}

int comm_p2p_begin(vpt_context* c, cudaStream_t stream) {
    if (!c->p2p_on) return VPT_OK;
    ++c->p2p_epoch;
    unsigned long long* fl[kMaxPeers];
    for (int p = 0; p < kMaxPeers; ++p) fl[p] = p < c->p2p_n ? p2p_flags(c->p2p_peer[p]) : nullptr;
    VPT_CU(c, launch_peer_signal(fl, c->p2p_n, c->rank, 0, c->p2p_epoch, stream));     // "my frame of the previous call has been consumed"
    c->launches++;
    return VPT_OK;
}

int comm_p2p_peers(vpt_context* c, cudaStream_t stream, PeerFrames* out) {
    *out = PeerFrames{};
    if (!c->p2p_on) return VPT_OK;
    VPT_CU(c, launch_peer_wait(p2p_flags(c->p2p_block), c->p2p_n, 0, c->p2p_epoch, stream));   // every peer has entered this call
    c->launches++;
    out->n = c->p2p_n;
    for (int p = 0; p < c->p2p_n; ++p) {
        char* base = reinterpret_cast<char*>(c->p2p_peer[p]);
        out->accum[p] = reinterpret_cast<float*>(base + kP2pHeader);
        out->display[p] = c->p2p_display ? reinterpret_cast<unsigned int*>(base + kP2pHeader + p2p_accum_bytes(c)) : nullptr;
    }
    return VPT_OK;
}

int comm_p2p_end(vpt_context* c, cudaStream_t stream) {
    if (!c->p2p_on) return VPT_OK;
    unsigned long long* fl[kMaxPeers];
    for (int p = 0; p < kMaxPeers; ++p) fl[p] = p < c->p2p_n ? p2p_flags(c->p2p_peer[p]) : nullptr;
    VPT_CU(c, launch_peer_signal(fl, c->p2p_n, c->rank, 1, c->p2p_epoch, stream));     // my stripes are in every frame ...
    VPT_CU(c, launch_peer_wait(p2p_flags(c->p2p_block), c->p2p_n, 1, c->p2p_epoch, stream));   // ... and everybody's are in mine
    c->launches += 2;
    return VPT_OK;
}

int comm_p2p_layers(vpt_context* c, const FrameGeom& g, const RenderRegion* rg, const LayerSources& src, cudaStream_t stream, const float3* motion) {
    if (!c->p2p_on || c->p2p_n < 2 || !c->p2p_layers) return VPT_OK;
    size_t off[kExchangeLayers], motion_off = 0;
    p2p_block_layout((size_t)c->p2p_w, (size_t)c->p2p_h, c->p2p_display, c->p2p_layers, c->p2p_slices, c->p2p_mattes, off, nullptr, &motion_off);
    if (c->p2p_layers & kPublishedLayers) {
        LayerPlanes dst;
        dst.n = c->p2p_n;
        for (int l = 0; l < kExchangeLayers; ++l)
            for (int p = 0; off[l] && p < c->p2p_n; ++p) dst.plane[l][p] = reinterpret_cast<float*>(reinterpret_cast<char*>(c->p2p_peer[p]) + off[l]);
        VPT_CU(c, launch_layers_publish(g, rg, src, dst, stream));
        c->launches++;
    }
    if (motion_off && motion) {
        // k_layers_publish with the motion vectors in the slot of a float3 layer and every other slot empty
        LayerSources ms;
        ms.src[XL_VOLUME] = reinterpret_cast<const float*>(motion);
        LayerPlanes dst;
        dst.n = c->p2p_n;
        for (int p = 0; p < c->p2p_n; ++p) dst.plane[XL_VOLUME][p] = reinterpret_cast<float*>(reinterpret_cast<char*>(c->p2p_peer[p]) + motion_off);
        VPT_CU(c, launch_layers_publish(g, rg, ms, dst, stream));
        c->launches++;
    }
    return VPT_OK;
}

int comm_p2p_binned(vpt_context* c, const FrameGeom& g, const RenderRegion* rg, const float4* deep, const float4* mattes, cudaStream_t stream) {
    if (!c->p2p_on || c->p2p_n < 2 || !(c->p2p_slices || c->p2p_mattes)) return VPT_OK;
    size_t off[kBinnedLayers];
    p2p_block_layout((size_t)c->p2p_w, (size_t)c->p2p_h, c->p2p_display, c->p2p_layers, c->p2p_slices, c->p2p_mattes, nullptr, off);
    const float4* src[kBinnedLayers] = {deep, mattes};
    const unsigned n[kBinnedLayers] = {c->p2p_slices, c->p2p_mattes};
    for (int b = 0; b < kBinnedLayers; ++b) {
        if (!n[b] || !src[b]) continue;                               // not exported / not active on this call: the arrays keep what they hold
        BinnedPlanes dst;
        dst.n = c->p2p_n;
        for (int p = 0; p < c->p2p_n; ++p) dst.plane[p] = reinterpret_cast<float4*>(reinterpret_cast<char*>(c->p2p_peer[p]) + off[b]);
        VPT_CU(c, launch_binned_publish(g, rg, src[b], (int)n[b], dst, stream));
        c->launches++;
    }
    return VPT_OK;
}

void comm_p2p_adapt_views(vpt_context* c, AdaptPeers* out, P2pAdaptLocal* local) {
    *out = AdaptPeers{};
    out->n = c->p2p_n;
    for (int p = 0; p < c->p2p_n; ++p) {
        char* base = reinterpret_cast<char*>(c->p2p_peer[p]);
        out->accum[p] = reinterpret_cast<float*>(base + kP2pHeader);
        out->display[p] = c->p2p_display ? reinterpret_cast<unsigned int*>(base + kP2pHeader + p2p_accum_bytes(c)) : nullptr;
        out->count[p] = reinterpret_cast<unsigned*>(base + p2p_count_offset(c));
        out->err[p] = reinterpret_cast<float*>(base + p2p_err_offset(c));
        out->tiles[p] = reinterpret_cast<unsigned*>(base + p2p_tiles_offset(c));
    }
    char* own = reinterpret_cast<char*>(c->p2p_block);
    local->halo = reinterpret_cast<const float*>(own + p2p_err_offset(c));
    local->tiles = reinterpret_cast<const unsigned*>(own + p2p_tiles_offset(c));
    local->error_word = p2p_flags(c->p2p_block) + 2 * kPeerFlagStride;
}

int comm_p2p_adapt_barrier(vpt_context* c, cudaStream_t stream) {
    ++c->p2p_adapt_epoch;
    unsigned long long* fl[kMaxPeers];
    for (int p = 0; p < kMaxPeers; ++p) fl[p] = p < c->p2p_n ? p2p_flags(c->p2p_peer[p]) : nullptr;
    VPT_CU(c, launch_peer_signal(fl, c->p2p_n, c->rank, kPeerFlagsAdapt, c->p2p_adapt_epoch, stream));
    VPT_CU(c, launch_peer_wait(p2p_flags(c->p2p_block), c->p2p_n, kPeerFlagsAdapt, c->p2p_adapt_epoch, stream));
    c->launches += 2;
    return VPT_OK;
}

} // namespace vpt

extern "C" {

int vpt_comm_p2p_export(vpt_context* c, int rank, int n_ranks, int stripe_rows, unsigned width, unsigned height, int with_display,
                        unsigned char handle_out[VPT_P2P_HANDLE_BYTES]) {
    return vpt_comm_p2p_export_layers(c, rank, n_ranks, stripe_rows, width, height, with_display, 0u, handle_out);
}

int vpt_comm_p2p_export_layers(vpt_context* c, int rank, int n_ranks, int stripe_rows, unsigned width, unsigned height, int with_display,
                               unsigned layers, unsigned char handle_out[VPT_P2P_HANDLE_BYTES]) {
    return vpt_comm_p2p_export_binned(c, rank, n_ranks, stripe_rows, width, height, with_display, layers, 0u, 0u, handle_out);
}

static_assert(vpt::kDeepMaxSlices == VPT_DEEP_MAX_SLICES && vpt::kMatteMax == VPT_MATTE_MAX, "binned layer limits");
// n_slices / n_mattes within 0..VPT_DEEP_MAX_SLICES / 0..VPT_MATTE_MAX; "" when they are
static std::string binned_count_error(unsigned n_slices, unsigned n_mattes) {
    if (n_slices > VPT_DEEP_MAX_SLICES)
        return "n_slices must be 0 or 1.." + std::to_string(VPT_DEEP_MAX_SLICES) + ", got " + std::to_string(n_slices);
    if (n_mattes > VPT_MATTE_MAX) return "n_mattes must be 0 or 1.." + std::to_string(VPT_MATTE_MAX) + ", got " + std::to_string(n_mattes);
    return "";
}

int vpt_comm_p2p_export_binned(vpt_context* c, int rank, int n_ranks, int stripe_rows, unsigned width, unsigned height, int with_display,
                               unsigned layers, unsigned n_slices, unsigned n_mattes, unsigned char handle_out[VPT_P2P_HANDLE_BYTES]) {
    if (!c || !handle_out || n_ranks < 1 || n_ranks > vpt::kMaxPeers || rank < 0 || rank >= n_ranks || stripe_rows < 1 || !width || !height)
        return vpt::fail_ctx(c, VPT_ERR_INVALID, "vpt_comm_p2p_export: bad arguments (at most 8 ranks: one NVSwitch domain)");
    if (layers & ~vpt::kLayerMask)
        return vpt::fail_ctx(c, VPT_ERR_INVALID, "vpt_comm_p2p_export_layers: unknown layer bits " + vpt::hex2(layers & ~vpt::kLayerMask));
    if (const std::string e = binned_count_error(n_slices, n_mattes); !e.empty())
        return vpt::fail_ctx(c, VPT_ERR_INVALID, "vpt_comm_p2p_export_binned: " + e);
    if (c->p2p_block) return vpt::fail_ctx(c, VPT_ERR_INVALID, "vpt_comm_p2p_export: already exported");
    static_assert(sizeof(cudaIpcMemHandle_t) == VPT_P2P_HANDLE_BYTES, "IPC handle size");
    static_assert(VPT_LAYER_DEPTH == 1u << vpt::XL_DEPTH && VPT_LAYER_ALPHA == 1u << vpt::XL_ALPHA && VPT_LAYER_VOLUME == 1u << vpt::XL_VOLUME &&
                  VPT_LAYER_SUN == 1u << vpt::XL_SUN && VPT_LAYER_POINT == 1u << vpt::XL_POINT && VPT_LAYER_EMISSION == 1u << vpt::XL_EMISSION &&
                  VPT_LAYER_ENVIRONMENT == 1u << vpt::XL_ENVIRONMENT, "layer bits");
    VPT_CU(c, cudaSetDevice(c->device));
    int rc = vpt_set_partition(c, rank, n_ranks, stripe_rows);
    if (rc != VPT_OK) return rc;
    VPT_CU(c, vpt::exchange_kernels_preload());
    c->p2p_w = (int)width; c->p2p_h = (int)height; c->p2p_display = with_display != 0; c->p2p_n = n_ranks; c->p2p_layers = layers;
    c->p2p_slices = n_slices; c->p2p_mattes = n_mattes;
    c->p2p_bytes = vpt::p2p_block_layout(width, height, c->p2p_display, layers, n_slices, n_mattes, nullptr);
    VPT_CU(c, cudaMalloc(&c->p2p_block, c->p2p_bytes));
    VPT_CU(c, cudaMemset(c->p2p_block, 0, c->p2p_bytes));
    const unsigned long long words[3] = {vpt::p2p_layout_word(c), vpt::p2p_binned_word(c), (unsigned long long)layers};
    static_assert(vpt::kP2pBinnedSlot == vpt::kP2pLayoutSlot + 1 && vpt::kP2pLayersSlot == vpt::kP2pLayoutSlot + 2,
                  "layout word, then the binned counts, then the layer mask");
    VPT_CU(c, cudaMemcpy(vpt::p2p_flags(c->p2p_block) + vpt::kP2pLayoutSlot, words, sizeof(words), cudaMemcpyHostToDevice));
    VPT_CU(c, cudaDeviceSynchronize());
    cudaIpcMemHandle_t h;
    VPT_CU(c, cudaIpcGetMemHandle(&h, c->p2p_block));
    memcpy(handle_out, &h, sizeof(h));
    return VPT_OK;
}

int vpt_comm_p2p_block_bytes(unsigned width, unsigned height, int with_display, unsigned layers, size_t* out) {
    if (!out || !width || !height) return vpt::fail_global(VPT_ERR_INVALID, "vpt_comm_p2p_block_bytes: bad arguments");
    if (layers & ~vpt::kLayerMask) return vpt::fail_global(VPT_ERR_INVALID, "vpt_comm_p2p_block_bytes: unknown layer bits");
    *out = vpt::p2p_block_layout(width, height, with_display != 0, layers, 0u, 0u, nullptr);
    return VPT_OK;
}

int vpt_comm_p2p_block_bytes_binned(unsigned width, unsigned height, int with_display, unsigned layers, unsigned n_slices, unsigned n_mattes,
                                    size_t* out) {
    if (!out || !width || !height) return vpt::fail_global(VPT_ERR_INVALID, "vpt_comm_p2p_block_bytes_binned: bad arguments");
    if (layers & ~vpt::kLayerMask) return vpt::fail_global(VPT_ERR_INVALID, "vpt_comm_p2p_block_bytes_binned: unknown layer bits");
    if (const std::string e = binned_count_error(n_slices, n_mattes); !e.empty())
        return vpt::fail_global(VPT_ERR_INVALID, "vpt_comm_p2p_block_bytes_binned: " + e);
    *out = vpt::p2p_block_layout(width, height, with_display != 0, layers, n_slices, n_mattes, nullptr);
    return VPT_OK;
}

int vpt_comm_p2p_binned(vpt_context* c, unsigned which, vpt_devptr_t* d_full, unsigned* k) {
    if (!c || !d_full || !c->p2p_block) return vpt::fail_ctx(c, VPT_ERR_INVALID, "vpt_comm_p2p_binned: no exchange block");
    if (which != VPT_BINNED_DEEP && which != VPT_BINNED_MATTES)
        return vpt::fail_ctx(c, VPT_ERR_INVALID, "vpt_comm_p2p_binned: " + std::to_string(which) + " is neither VPT_BINNED_DEEP nor VPT_BINNED_MATTES");
    const int b = which == VPT_BINNED_DEEP ? vpt::BL_DEEP : vpt::BL_MATTES;
    const unsigned n = b == vpt::BL_DEEP ? c->p2p_slices : c->p2p_mattes;
    if (!n)
        return vpt::fail_ctx(c, VPT_ERR_INVALID, std::string("vpt_comm_p2p_binned: the block was exported without ") +
                                                 (b == vpt::BL_DEEP ? "deep slices" : "mattes") + " (vpt_comm_p2p_export_binned)");
    size_t off[vpt::kBinnedLayers];
    vpt::p2p_block_layout((size_t)c->p2p_w, (size_t)c->p2p_h, c->p2p_display, c->p2p_layers, c->p2p_slices, c->p2p_mattes, nullptr, off);
    *d_full = (vpt_devptr_t)(reinterpret_cast<char*>(c->p2p_block) + off[b]);
    if (k) *k = n;
    return VPT_OK;
}

int vpt_comm_p2p_layer(vpt_context* c, unsigned layer, vpt_devptr_t* d_full) {
    if (!c || !d_full || !c->p2p_block) return vpt::fail_ctx(c, VPT_ERR_INVALID, "vpt_comm_p2p_layer: no exchange block");
    int l = 0;
    while (l < vpt::kExchangeLayers && layer != 1u << l) ++l;
    if (l == vpt::kExchangeLayers && layer != vpt::kMotionLayerBit)
        return vpt::fail_ctx(c, VPT_ERR_INVALID, "vpt_comm_p2p_layer: " + std::to_string(layer) + " is not one VPT_LAYER_* bit");
    if (!(c->p2p_layers & layer))
        return vpt::fail_ctx(c, VPT_ERR_INVALID, "vpt_comm_p2p_layer: the block was exported without layer " + std::to_string(layer) + " (vpt_comm_p2p_export_layers)");
    size_t off[vpt::kExchangeLayers], motion_off = 0;
    vpt::p2p_block_layout((size_t)c->p2p_w, (size_t)c->p2p_h, c->p2p_display, c->p2p_layers, c->p2p_slices, c->p2p_mattes, off, nullptr, &motion_off);
    *d_full = (vpt_devptr_t)(reinterpret_cast<char*>(c->p2p_block) + (l < vpt::kExchangeLayers ? off[l] : motion_off));
    return VPT_OK;
}

int vpt_comm_p2p_import(vpt_context* c, const unsigned char* handles) {
    if (!c || !handles || !c->p2p_block) return vpt::fail_ctx(c, VPT_ERR_INVALID, "vpt_comm_p2p_import: call vpt_comm_p2p_export first");
    for (int p = 0; p < c->p2p_n; ++p) {
        if (p == c->rank) { c->p2p_peer[p] = c->p2p_block; continue; }
        cudaIpcMemHandle_t h; memcpy(&h, handles + (size_t)p * VPT_P2P_HANDLE_BYTES, sizeof(h));
        VPT_CU(c, cudaIpcOpenMemHandle(&c->p2p_peer[p], h, cudaIpcMemLazyEnablePeerAccess));
    }
    if (int rc = vpt::p2p_check_layouts(c, "vpt_comm_p2p_import"); rc != VPT_OK) {
        for (int p = 0; p < c->p2p_n; ++p) { if (p != c->rank && c->p2p_peer[p]) cudaIpcCloseMemHandle(c->p2p_peer[p]); c->p2p_peer[p] = nullptr; }
        return rc;
    }
    c->p2p_on = true; c->p2p_epoch = 0; c->p2p_adapt_epoch = 0;
    return VPT_OK;
}

int vpt_comm_p2p_import_local(vpt_context* c, const vpt_devptr_t* blocks) {
    if (!c || !blocks || !c->p2p_block) return vpt::fail_ctx(c, VPT_ERR_INVALID, "vpt_comm_p2p_import_local: call vpt_comm_p2p_export first");
    for (int p = 0; p < c->p2p_n; ++p) {
        if (p != c->rank && !blocks[p]) return vpt::fail_ctx(c, VPT_ERR_INVALID, "vpt_comm_p2p_import_local: null block");
        c->p2p_peer[p] = p == c->rank ? c->p2p_block : reinterpret_cast<void*>(blocks[p]);
    }
    if (int rc = vpt::p2p_check_layouts(c, "vpt_comm_p2p_import_local"); rc != VPT_OK) {
        for (auto& q : c->p2p_peer) q = nullptr;
        return rc;
    }
    c->p2p_local = true; c->p2p_on = true; c->p2p_epoch = 0; c->p2p_adapt_epoch = 0;
    return VPT_OK;
}

int vpt_comm_p2p_block(vpt_context* c, vpt_devptr_t* d_block) {
    if (!c || !d_block || !c->p2p_block) return vpt::fail_ctx(c, VPT_ERR_INVALID, "vpt_comm_p2p_block: no exchange block");
    *d_block = (vpt_devptr_t)c->p2p_block;
    return VPT_OK;
}

int vpt_comm_p2p_frame(vpt_context* c, vpt_devptr_t* d_full_accum, vpt_devptr_t* d_full_display) {
    if (!c || !c->p2p_block) return vpt::fail_ctx(c, VPT_ERR_INVALID, "vpt_comm_p2p_frame: no exchange block");
    char* base = reinterpret_cast<char*>(c->p2p_block);
    if (d_full_accum) *d_full_accum = (vpt_devptr_t)(base + vpt::kP2pHeader);
    if (d_full_display) *d_full_display = c->p2p_display ? (vpt_devptr_t)(base + vpt::kP2pHeader + vpt::p2p_accum_bytes(c)) : 0;
    return VPT_OK;
}

int vpt_comm_p2p_adaptive_frame(vpt_context* c, vpt_devptr_t* d_full_pass_count, vpt_devptr_t* d_full_rel_error) {
    if (!c || !c->p2p_block) return vpt::fail_ctx(c, VPT_ERR_INVALID, "vpt_comm_p2p_adaptive_frame: no exchange block");
    char* base = reinterpret_cast<char*>(c->p2p_block);
    if (d_full_pass_count) *d_full_pass_count = (vpt_devptr_t)(base + vpt::p2p_count_offset(c));
    if (d_full_rel_error) *d_full_rel_error = (vpt_devptr_t)(base + vpt::p2p_err_offset(c));
    return VPT_OK;
}

int vpt_comm_p2p_enable(vpt_context* c, int on) {
    if (!c || !c->p2p_block || !c->p2p_peer[c->rank]) return vpt::fail_ctx(c, VPT_ERR_INVALID, "vpt_comm_p2p_enable: exchange not set up");
    c->p2p_on = on != 0;
    return VPT_OK;
}

int vpt_comm_p2p_status(vpt_context* c, unsigned long long* timeouts) {
    if (!c || !timeouts || !c->p2p_block) return vpt::fail_ctx(c, VPT_ERR_INVALID, "vpt_comm_p2p_status: no exchange block");
    VPT_CU(c, cudaMemcpy(timeouts, vpt::p2p_flags(c->p2p_block) + 2 * vpt::kPeerFlagStride, sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    return VPT_OK;
}

int vpt_comm_get_unique_id(unsigned char id_out[VPT_COMM_ID_BYTES]) {
    if (!id_out) return vpt::fail_global(VPT_ERR_INVALID, "vpt_comm_get_unique_id: null argument");
    NcclApi& n = nccl();
    if (!n.error.empty()) return vpt::fail_global(VPT_ERR_UNSUPPORTED, "vpt_comm_get_unique_id: " + n.error);
    nccl_unique_id id; memset(&id, 0, sizeof(id));
    nccl_result_t r = n.GetUniqueId(&id);
    if (r != 0) return vpt::fail_global(VPT_ERR_CUDA, std::string("ncclGetUniqueId: ") + n.GetErrorString(r));
    memcpy(id_out, id.internal, VPT_COMM_ID_BYTES);
    return VPT_OK;
}

int vpt_comm_init(vpt_context* c, const unsigned char id[VPT_COMM_ID_BYTES], int rank, int n_ranks, int stripe_rows) {
    if (!c || !id || n_ranks < 1 || rank < 0 || rank >= n_ranks || stripe_rows < 1) return vpt::fail_ctx(c, VPT_ERR_INVALID, "vpt_comm_init: bad arguments");
    if (c->nccl_comm) return vpt::fail_ctx(c, VPT_ERR_INVALID, "vpt_comm_init: communicator already initialised");
    NcclApi& n = nccl();
    if (!n.error.empty()) return vpt::fail_ctx(c, VPT_ERR_UNSUPPORTED, "vpt_comm_init: " + n.error);
    VPT_CU(c, cudaSetDevice(c->device));
    nccl_unique_id uid; memcpy(uid.internal, id, VPT_COMM_ID_BYTES);
    nccl_comm_t comm = nullptr;
    nccl_result_t r = n.CommInitRank(&comm, n_ranks, uid, rank);
    if (r != 0) return nccl_fail(c, "ncclCommInitRank", r);
    c->nccl_comm = comm;
    VPT_CU(c, cudaStreamCreateWithFlags(&c->comm_stream, cudaStreamNonBlocking));
    VPT_CU(c, cudaEventCreateWithFlags(&c->ev_render_done, cudaEventDisableTiming));
    VPT_CU(c, cudaEventCreateWithFlags(&c->ev_gather_done, cudaEventDisableTiming));
    return vpt_set_partition(c, rank, n_ranks, stripe_rows);
}

int vpt_comm_set_gather(vpt_context* c, void* d_full_accum, void* d_full_display) {
    if (!c) return VPT_ERR_INVALID;
    if ((d_full_accum || d_full_display) && !c->nccl_comm) return vpt::fail_ctx(c, VPT_ERR_INVALID, "vpt_comm_set_gather: call vpt_comm_init first");
    c->d_full_accum = d_full_accum; c->d_full_display = d_full_display;
    return VPT_OK;
}

int vpt_comm_wait(vpt_context* c, void* stream) {
    if (!c) return VPT_ERR_INVALID;
    return vpt::comm_before_accum_write(c, (cudaStream_t)stream);
}

int vpt_comm_info(vpt_context* c, int* nccl_version, int* rank, int* n_ranks) {
    if (!c) return VPT_ERR_INVALID;
    NcclApi& n = nccl();
    if (nccl_version) { int v = 0; if (n.GetVersion) n.GetVersion(&v); *nccl_version = v; }
    if (rank) *rank = c->rank;
    if (n_ranks) *n_ranks = c->nccl_comm ? c->n_ranks : 1;
    return VPT_OK;
}

int vpt_comm_destroy(vpt_context* c) {
    if (!c) return VPT_ERR_INVALID;
    if (c->nccl_comm) {
        if (c->comm_stream) cudaStreamSynchronize(c->comm_stream);
        nccl().CommDestroy((nccl_comm_t)c->nccl_comm); c->nccl_comm = nullptr;
    }
    if (c->comm_stream) { cudaStreamDestroy(c->comm_stream); c->comm_stream = nullptr; }
    if (c->ev_render_done) { cudaEventDestroy(c->ev_render_done); c->ev_render_done = nullptr; }
    if (c->ev_gather_done) { cudaEventDestroy(c->ev_gather_done); c->ev_gather_done = nullptr; }
    cudaFree(c->d_gathered); c->d_gathered = nullptr; c->cap_gathered = 0;
    cudaFree(c->d_gathered_disp); c->d_gathered_disp = nullptr; c->cap_gathered_disp = 0;
    c->d_full_accum = c->d_full_display = nullptr; c->gather_pending = false;
    if (c->p2p_block) {
        cudaDeviceSynchronize();
        if (!c->p2p_local) for (int p = 0; p < c->p2p_n; ++p) if (p != c->rank && c->p2p_peer[p]) cudaIpcCloseMemHandle(c->p2p_peer[p]);
        cudaFree(c->p2p_block); c->p2p_block = nullptr; c->p2p_on = false; c->p2p_n = 0; c->p2p_layers = 0; c->p2p_slices = c->p2p_mattes = 0;
        for (auto& q : c->p2p_peer) q = nullptr;
    }
    return VPT_OK;
}

} // extern "C"
