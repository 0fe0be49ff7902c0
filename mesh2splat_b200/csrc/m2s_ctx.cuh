// m2s_ctx.cuh — the context and the device scene behind the C ABI's handles, and the host internals that more than one of
// m2s_api.cu (context), m2s_scene.cu (device scene), m2s_convert.cu (conversion) and m2s_viewer.cu (viewer passes) use.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include "m2s_device.cuh"
#include "m2s_host.h"

#define CUDA_TRY(expr)                                                                              \
    do {                                                                                            \
        cudaError_t _e = (expr);                                                                    \
        if (_e != cudaSuccess) {                                                                    \
            m2s::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));                     \
            return (_e == cudaErrorNoDevice || _e == cudaErrorInsufficientDriver) ? M2S_E_NOGPU : M2S_E_CUDA; \
        }                                                                                           \
    } while (0)

namespace m2s {

struct Scratch {           // a device buffer the context owns and grows on demand (grow); m2s_ctx_destroy frees it
    void* p = nullptr;
    size_t bytes = 0;
};
// scratch of one binned pass (the splat draw, the cube raster, the mesh depth pre-pass): per-item counts and tile ranges
// (BinLayout, m2s_bin.cuh), and the pair sort (SortLayout, m2s_sort.cuh)
struct BinScratch {
    Scratch bins, pairs;
};
struct VRangeSlot {        // v-range reduction of one pipeline chunk: device buffer + pinned host copy + "copy done" event
    int* d_minmax = nullptr;     // [2 * ntex]: sortable-int min | max of v per texture, then 1 non-finite flag (armed: see vrange_publish_kernel)
    int* h_minmax = nullptr;     // pinned + mapped: written by the publish kernel, followed (8-byte aligned) by the tag
    int* h_minmax_dev = nullptr; // its device view
    unsigned long long* h_tag = nullptr;      // host view of the tag
    unsigned long long* h_tag_dev = nullptr;
    unsigned long long tag = 0;               // the tag the current reduction will publish
    cudaEvent_t ev = nullptr;    // recorded behind the publish kernel (error path: a failed launch never writes the tag)
};

}  // namespace m2s

struct m2s_ctx {
    int device = 0;
    int sm_count = 0;
    cudaStream_t stream = nullptr;
    uint32_t* d_sched = nullptr;             // 8 x 128 B (one scheduler word per cache line)
    unsigned long long* d_counter = nullptr; // running fragment counter
    unsigned long long* d_total = nullptr;   // published count
    uint32_t* d_nitems = nullptr;            // work items queued by the last raster launch
    uint32_t* d_prepass_valid = nullptr;     // counter of the synchronous m2s_prepass
    unsigned long long* h_total = nullptr;   // pinned
    uint32_t* h_status = nullptr;            // pinned + mapped: raised by device-side waits that timed out (fused gather)
    uint32_t* d_status = nullptr;            // its device view
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev_mid = nullptr;
    // convert_host pipeline: a second stream for the downloads, per-chunk counts and events
    static constexpr int kMaxChunks = 8;
    cudaStream_t stream2 = nullptr;
    cudaStream_t stream3 = nullptr;              // uploads of the host pipeline: the copy engine keeps going while chunk kernels run
    cudaStream_t up = nullptr;                   // stream triangle chunks are uploaded on (= stream, or stream3 inside the pipeline)
    // the host pipeline keeps TWO copy engines busy in the upload direction (two streams deliver more than one:
    // scripts/pcie_probe.py measures it) and never puts a kernel between two copies of a stream (a copy behind a kernel of
    // its own stream waits for it: with the v-range and mip kernels on the copy stream every chunk cost ~40 us of bubbles)
    cudaStream_t stream4 = nullptr;              // texture rows
    cudaStream_t stream5 = nullptr;              // v-range reductions and their 8-byte results
    cudaStream_t tex_up = nullptr;               // stream texture rows are uploaded on (= up, or stream4 inside the pipeline)
    cudaStream_t mip = nullptr;                  // stream their mip rows are generated on (= tex_up, or the compute stream inside the pipeline)
    cudaStream_t aux = nullptr;                  // stream the v-range reductions run on (= up, or stream5 inside the pipeline)
    cudaEvent_t ev_tri[kMaxChunks] = {};         // "chunk c's triangles are resident"
    cudaEvent_t ev_up[kMaxChunks] = {};          // "chunk c's texture rows are resident"
    cudaEvent_t ev_alloc = nullptr;
    unsigned long long* d_chunk_tot = nullptr;   // [kMaxChunks]
    unsigned long long* h_chunk_tot = nullptr;   // pinned + mapped: {count, tag} per chunk, written by the raster kernel
    unsigned long long host_seq = 0;             // tag generator
    // file writer: two pinned staging buffers (download of block i overlaps the write of block i-1)
    static constexpr size_t kStageBytes = 32u << 20;
    unsigned char* h_stage[2] = {nullptr, nullptr};
    cudaEvent_t ev_chunk[kMaxChunks] = {};
    m2s::VRangeSlot vr[kMaxChunks];          // v-range reductions of the host pipeline (lazy texture upload)
    uint32_t vr_ntex = 0;                    // textures the slots are sized for
    bool vr_dirty = false;                   // a pipeline was abandoned half way: the device copies must be re-armed
    static constexpr int kLayouts = 5;
    int blocks_per_sm[kLayouts] = {};       // raster kernel (persistent)
    int frag_blocks_per_sm[kLayouts] = {};  // fragment kernel
    unsigned long long epoch = 0;            // pairs up the ranks' calls of the fused gather
    bool dirty = true;                       // scheduler state needs a memset before the next launch
    // scratch owned by the context (grown on demand)
    m2s::Scratch out, keys;                  // convert_host output and keys
    m2s::Scratch trifrag, items;             // between the raster and the fragment kernel: TriRec per triangle, FragItem queue
    m2s::Scratch sort;                       // depth sort: control words, alternate key and value buffers (SortLayout, m2s_sort.cuh)
    m2s::BinScratch splat_bins, shadow_bins, depth_bins;  // the binned passes: splat draw, cube raster, mesh depth pre-pass
    m2s::Scratch light_quads;                // shadow pass: light records when the caller passes none
    m2s::Scratch ply_rows;                   // .ply reader: two slots of one block of raw vertex rows (m2s_ply_read.cu)
    // every Scratch above (m2s_ctx_destroy frees them): a member added above is added here too
    std::vector<m2s::Scratch*> all_scratch() {
        return {&out, &keys, &trifrag, &items, &sort, &light_quads, &ply_rows, &splat_bins.bins, &splat_bins.pairs, &shadow_bins.bins,
                &shadow_bins.pairs, &depth_bins.bins, &depth_bins.pairs};
    }
    uint64_t ply_h2d = 0;                    // row bytes m2s_ply_read copied host -> device
};

struct m2s_dscene {
    float4* d_tris = nullptr;
    uint64_t ntri = 0;
    m2s::DRange* d_ranges = nullptr;
    uint32_t nranges = 0;
    m2s::DPrim* d_prims = nullptr;
    uint32_t nprims = 0;
    m2s::DTexture* d_texs = nullptr;
    uint32_t* d_arena = nullptr;  // all mip chains of all textures
    uint32_t ntex = 0;
    std::vector<m2s::DTexture> h_texs;
    std::vector<void*> allocs;
    // lazily uploaded textures (host pipeline): level-0 rows travel in groups of kTexGroupRows rows, each group brings
    // its own rows of the mip levels 1..4 with it (a group of 16 rows is closed under the 2x2 box filter)
    std::vector<const uint8_t*> h_rgba;              // host images (valid for the duration of the call that uploads lazily)
    std::vector<std::vector<uint8_t>> present;       // per texture, per row group: already on the device
    uint64_t h2d_bytes = 0;                          // payload copied host -> device for this scene so far
};

namespace m2s {

// Context scratch grows on the stream that will USE it: the free of the old block is ordered after the kernels
// already enqueued there, the new block is ready before the next one.  (A caller that alternates between streams
// without synchronising them must not share one context: documented in m2s.h.)
inline m2s_status grow(m2s_ctx* ctx, Scratch& s, size_t need, cudaStream_t stream = nullptr) {
    if (s.bytes >= need) return M2S_OK;
    if (!stream) stream = ctx->stream;
    if (s.p) CUDA_TRY(cudaFreeAsync(s.p, stream));
    s.p = nullptr; s.bytes = 0;
    CUDA_TRY(cudaMallocAsync(&s.p, need + need / 4, stream));  // 25 % head room: density sweeps do not reallocate at every step
    s.bytes = need + need / 4;
    return M2S_OK;
}

// the caller's stream of an enqueue entry point, the context's when it passes none
inline cudaStream_t pick_stream(const m2s_ctx* ctx, void* stream) { return stream ? (cudaStream_t)stream : ctx->stream; }

// the triangles [first, first + count) of a list of n: first clamped to n, count 0 or past the end = the rest of the list
struct TriRange { uint64_t first, count; };
inline TriRange tri_range(uint64_t first, uint64_t count, uint64_t n) {
    first = std::min(first, n);
    if (count == 0 || first + count > n) count = n - first;
    return {first, count};
}

// ---- argument checks (the viewer's own: m2s_viewer.cu) ----
// M2S_E_INVALID with the error "<fn>: <msg>"
inline m2s_status invalid(const char* fn, const std::string& msg) { set_error(fn + (": " + msg)); return M2S_E_INVALID; }
// every pointer a multiple of its alignment; otherwise false, with the error "<fn>: <msg>"
struct Aligned { const void* p; uintptr_t bytes; };
inline bool aligned_ok(const char* fn, const char* msg, std::initializer_list<Aligned> v) {
    for (const Aligned& a : v)
        if (reinterpret_cast<uintptr_t>(a.p) & (a.bytes - 1)) { invalid(fn, msg); return false; }
    return true;
}

// ---- the device scene (m2s_scene.cu) ----
constexpr uint32_t kTexGroupRows = 16;               // = 2^M2S_MAX_MIP_LEVEL
struct MipRun { uint32_t t, g0, g1; };   // levels 1.. of the row groups [g0, g1) of texture t are still to be generated

// first_tris < triangle_count: only that many triangles are copied here (the caller streams the rest into
// d_tris itself, interleaved with its launches) and the stream is not synchronised.
// lazy_tex: the images are NOT copied here; the caller brings in the row groups its triangle ranges sample with
// vrange_enqueue + upload_groups_from_vrange (m2s_convert_host pipelines them with the triangle chunks,
// m2s_scene_upload_range uploads what one shard needs).
m2s_status scene_upload_impl(m2s_ctx* ctx, const m2s_scene* sc, m2s_dscene** out, uint64_t first_tris, bool sync,
                             uint64_t tri_offset = 0, bool lazy_tex = false);
// enqueue on ctx->aux: reduce the v-range of triangles [lo, hi) (already on the device) per texture, copy it to the
// slot's pinned buffer, record the slot's event
m2s_status vrange_enqueue(m2s_ctx* ctx, m2s_dscene* d, uint64_t lo, uint64_t hi, int slot);
// rows [g0, g1) x kTexGroupRows of texture t go up; their mip rows are generated, or appended to *deferred
m2s_status upload_texture_groups(m2s_ctx* ctx, m2s_dscene* d, uint32_t t, uint32_t g0, uint32_t g1, std::vector<MipRun>* deferred = nullptr);

// Which texture rows can the triangles [lo, hi) sample?  The v-range per texture is reduced ON THE GPU from the triangles
// already uploaded (vrange_launch: the host would have to stream the same 144 B/triangle through one core — ~1 ms for
// the bench scene), copied back (8 bytes per texture) and turned into 16-row groups here: +-3 groups cover the
// footprints of all five mip levels (level l reaches 2^(l+1) level-0 rows beyond the sample point, plus the drift of
// non-power-of-two chains) and the REPEAT wrap at both ends; a range whose v spans a whole period (or is not finite)
// takes the whole image.
// `idle` (optional) is called while the host waits for the reduction: the host pipeline enqueues ready downloads there
inline float sortable_to_float(int i) { i ^= (i >> 31) & 0x7fffffff; float f; std::memcpy(&f, &i, 4); return f; }
template <class Idle>
m2s_status upload_groups_from_vrange(m2s_ctx* ctx, m2s_dscene* d, int slot, Idle idle, std::vector<MipRun>* deferred = nullptr) {
    const uint32_t nt = d->ntex;
    if (!nt) return M2S_OK;
    for (uint32_t spin = 0;; ++spin) {
        if (__atomic_load_n(ctx->vr[slot].h_tag, __ATOMIC_ACQUIRE) == ctx->vr[slot].tag) break;   // the values are ordered before the tag
        if ((spin & 255u) == 255u) {  // a failed launch never writes the tag: ask the stream now and then
            const cudaError_t q = cudaEventQuery(ctx->vr[slot].ev);
            if (q == cudaSuccess) { if (__atomic_load_n(ctx->vr[slot].h_tag, __ATOMIC_ACQUIRE) == ctx->vr[slot].tag) break; }
            else if (q != cudaErrorNotReady) { set_error(std::string("v-range reduction: ") + cudaGetErrorString(q)); return M2S_E_CUDA; }
        }
        const cudaError_t ie = idle();
        if (ie != cudaSuccess) { set_error(std::string("convert_host download: ") + cudaGetErrorString(ie)); return M2S_E_CUDA; }
    }
    const int* mm = ctx->vr[slot].h_minmax;
    const bool finite = mm[2 * nt] == 0;
    for (uint32_t t = 0; t < nt; ++t) {
        if (mm[t] > mm[nt + t]) continue;  // no triangle of the range samples this texture
        const uint32_t ng = (uint32_t)d->present[t].size();
        std::vector<uint8_t> need(ng, 0);
        const float vmin = sortable_to_float(mm[t]), vmax = sortable_to_float(mm[nt + t]);
        const float fl = std::floor(vmin);
        if (!finite || !(vmax - fl <= 1.0f) || ng <= 8) std::fill(need.begin(), need.end(), 1);  // v = 1.0 exactly wraps to the first rows (modulo below)
        else {
            const float H = (float)d->h_texs[t].h[0];
            const long long ra = (long long)std::floor((vmin - fl) * H) - 1, rb = (long long)std::floor((vmax - fl) * H) + 1;
            const long long ga = ra / (long long)kTexGroupRows - 3 - (ra < 0), gb = rb / (long long)kTexGroupRows + 3;
            if (gb - ga + 1 >= (long long)ng) std::fill(need.begin(), need.end(), 1);
            else for (long long g = ga; g <= gb; ++g) need[(size_t)(((g % ng) + ng) % ng)] = 1;  // REPEAT: wraps at both ends
        }
        for (uint32_t g = 0; g < ng;) {
            if (!need[g] || d->present[t][g]) { ++g; continue; }
            uint32_t e = g;
            while (e < ng && need[e] && !d->present[t][e]) ++e;
            m2s_status st = upload_texture_groups(ctx, d, t, g, e, deferred);
            if (st != M2S_OK) return st;
            g = e;
        }
    }
    return M2S_OK;
}

// Upload only the maps a layout consumes: PACKED56 carries neither normal nor metallic/roughness, the
// standard .ply row no metallic/roughness — their texels would cross PCIe for nothing.
struct SlimScene {
    std::vector<m2s_primitive> prims;
    std::vector<m2s_texture> texs;
    m2s_scene scene;
    SlimScene(const m2s_scene* sc, uint32_t layout) : prims(sc->primitives, sc->primitives + sc->primitive_count), scene(*sc) {
        const bool need_normal = layout != M2S_LAYOUT_PACKED56;
        const bool need_mr = layout == M2S_LAYOUT_REF96 || layout == M2S_LAYOUT_PLY_PBR || layout == M2S_LAYOUT_PLY_COMPRESSED;
        std::vector<int32_t> remap(sc->texture_count, -1);
        auto use = [&](int32_t& idx, bool needed) {
            if (idx < 0 || !needed || (uint32_t)idx >= sc->texture_count) { if (idx >= 0 && (uint32_t)idx < sc->texture_count) idx = -1; return; }
            if (remap[idx] < 0) { remap[idx] = (int32_t)texs.size(); texs.push_back(sc->textures[idx]); }
            idx = remap[idx];
        };
        for (auto& pr : prims) { use(pr.albedo_texture, true); use(pr.normal_texture, need_normal); use(pr.metallic_roughness_texture, need_mr); }
        scene.primitives = prims.data();
        scene.textures = texs.data();
        scene.texture_count = (uint32_t)texs.size();
    }
};

// ---- the conversion (m2s_convert.cu) ----
// the records a conversion stores: max_gaussians, else the reference's rule (out_capacity if uncapped), <= out_capacity
uint64_t effective_cap(const m2s_dscene* s, const m2s_params* p, uint64_t out_capacity);
m2s_status convert_enqueue_impl(m2s_ctx* ctx, const m2s_dscene* s, const m2s_params* p, void* d_out, uint64_t out_capacity,
                                uint64_t* d_keys, uint64_t* d_total, void* stream_, const m2s_peers* peers,
                                const unsigned long long* prev_totals = nullptr, uint32_t nprev = 0,
                                unsigned long long* host_total = nullptr, unsigned long long host_tag = 0, cudaEvent_t mid = nullptr);

}  // namespace m2s
