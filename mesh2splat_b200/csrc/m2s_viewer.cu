// m2s_viewer.cu — C-ABI implementation (include/m2s.h): the viewer's passes.  Prepass, depth sort, splat draw, shadow
// map, deferred lighting and mesh depth pre-pass: argument checks, the uniforms built on the host, and the launches.
#include <cmath>

#include "m2s_bin.cuh"
#include "m2s_ctx.cuh"
#include "m2s_depth.cuh"
#include "m2s_light.cuh"
#include "m2s_prepass.cuh"
#include "m2s_sort.cuh"
#include "m2s_splat.cuh"

using namespace m2s;

// ---- argument checks shared by the passes: false, with the error "<fn>: <message>", when a value is out of range ----
// every value in 1..max: "<names> must be 1..<max>"
static bool sizes_ok(const char* fn, const char* names, uint32_t max, std::initializer_list<uint32_t> v) {
    for (uint32_t x : v)
        if (x < 1 || x > max) { invalid(fn, std::string(names) + " must be 1.." + std::to_string(max)); return false; }
    return true;
}
// a pair budget the pair sort can take
static bool pair_budget_ok(const char* fn, uint64_t max_pairs) {
    if (max_pairs >= kSplatMaxPairs) { invalid(fn, "max_pairs too large (< 2^30 supported)"); return false; }
    return true;
}

// ---- the viewer prepass (SURVEY 8 f-4): GaussiansPrepass::execute + gaussianSplattingPrepassCS.glsl ----------------
static bool invert4(const double m[16], double inv[16]) {   // column-major, cofactors
    inv[0] = m[5] * m[10] * m[15] - m[5] * m[11] * m[14] - m[9] * m[6] * m[15] + m[9] * m[7] * m[14] + m[13] * m[6] * m[11] - m[13] * m[7] * m[10];
    inv[4] = -m[4] * m[10] * m[15] + m[4] * m[11] * m[14] + m[8] * m[6] * m[15] - m[8] * m[7] * m[14] - m[12] * m[6] * m[11] + m[12] * m[7] * m[10];
    inv[8] = m[4] * m[9] * m[15] - m[4] * m[11] * m[13] - m[8] * m[5] * m[15] + m[8] * m[7] * m[13] + m[12] * m[5] * m[11] - m[12] * m[7] * m[9];
    inv[12] = -m[4] * m[9] * m[14] + m[4] * m[10] * m[13] + m[8] * m[5] * m[14] - m[8] * m[6] * m[13] - m[12] * m[5] * m[10] + m[12] * m[6] * m[9];
    inv[1] = -m[1] * m[10] * m[15] + m[1] * m[11] * m[14] + m[9] * m[2] * m[15] - m[9] * m[3] * m[14] - m[13] * m[2] * m[11] + m[13] * m[3] * m[10];
    inv[5] = m[0] * m[10] * m[15] - m[0] * m[11] * m[14] - m[8] * m[2] * m[15] + m[8] * m[3] * m[14] + m[12] * m[2] * m[11] - m[12] * m[3] * m[10];
    inv[9] = -m[0] * m[9] * m[15] + m[0] * m[11] * m[13] + m[8] * m[1] * m[15] - m[8] * m[3] * m[13] - m[12] * m[1] * m[11] + m[12] * m[3] * m[9];
    inv[13] = m[0] * m[9] * m[14] - m[0] * m[10] * m[13] - m[8] * m[1] * m[14] + m[8] * m[2] * m[13] + m[12] * m[1] * m[10] - m[12] * m[2] * m[9];
    inv[2] = m[1] * m[6] * m[15] - m[1] * m[7] * m[14] - m[5] * m[2] * m[15] + m[5] * m[3] * m[14] + m[13] * m[2] * m[7] - m[13] * m[3] * m[6];
    inv[6] = -m[0] * m[6] * m[15] + m[0] * m[7] * m[14] + m[4] * m[2] * m[15] - m[4] * m[3] * m[14] - m[12] * m[2] * m[7] + m[12] * m[3] * m[6];
    inv[10] = m[0] * m[5] * m[15] - m[0] * m[7] * m[13] - m[4] * m[1] * m[15] + m[4] * m[3] * m[13] + m[12] * m[1] * m[7] - m[12] * m[3] * m[5];
    inv[14] = -m[0] * m[5] * m[14] + m[0] * m[6] * m[13] + m[4] * m[1] * m[14] - m[4] * m[2] * m[13] - m[12] * m[1] * m[6] + m[12] * m[2] * m[5];
    inv[3] = -m[1] * m[6] * m[11] + m[1] * m[7] * m[10] + m[5] * m[2] * m[11] - m[5] * m[3] * m[10] - m[9] * m[2] * m[7] + m[9] * m[3] * m[6];
    inv[7] = m[0] * m[6] * m[11] - m[0] * m[7] * m[10] - m[4] * m[2] * m[11] + m[4] * m[3] * m[10] + m[8] * m[2] * m[7] - m[8] * m[3] * m[6];
    inv[11] = -m[0] * m[5] * m[11] + m[0] * m[7] * m[9] + m[4] * m[1] * m[11] - m[4] * m[3] * m[9] - m[8] * m[1] * m[7] + m[8] * m[3] * m[5];
    inv[15] = m[0] * m[5] * m[10] - m[0] * m[6] * m[9] - m[4] * m[1] * m[10] + m[4] * m[2] * m[9] + m[8] * m[1] * m[6] - m[8] * m[2] * m[5];
    const double det = m[0] * inv[0] + m[1] * inv[4] + m[2] * inv[8] + m[3] * inv[12];
    if (det == 0.0) return false;
    for (int k = 0; k < 16; ++k) inv[k] /= det;
    return true;
}

// the `layout` of m2s_prepass* / m2s_shadow_map*: the record layout and the reference's u_format / u_plyHasPbr it stands for
struct ViewInput { uint32_t layout, fmt, ply_has_pbr; };
static bool view_input(uint32_t layout, ViewInput& v) {
    switch (layout) {
        case M2S_LAYOUT_REF96: v = {0u, 0u, 0u}; return true;     // a conversion's records
        case M2S_LAYOUT_PACKED56: v = {1u, 1u, 0u}; return true;  // a standard 3DGS gaussian, u_format 1 without PBR values
        case M2S_VIEW_PLY: v = {0u, 1u, 0u}; return true;         // REF96 records as m2s_ply_read loads them
        case M2S_VIEW_PLY_PBR: v = {0u, 1u, 1u}; return true;
        default: return false;
    }
}

// d_valid: the enqueue forms' counter (the synchronous forms use the context's, never NULL)
static m2s_status prepass_check(const m2s_ctx* ctx, const void* d_records, uint64_t count, const m2s_prepass_params* p, const void* d_quads,
                                const float* d_depths, bool has_valid) {
    const char* fn = "m2s_prepass";
    if (!ctx || !p || !has_valid || (count && (!d_records || !d_quads || !d_depths))) return invalid(fn, "NULL argument");
    ViewInput v;
    if (!view_input(p->layout, v)) return invalid(fn, "layouts REF96, PACKED56, VIEW_PLY and VIEW_PLY_PBR only");
    if (p->render_mode == 3 || (p->render_mode > 2 && p->render_mode != 6)) return invalid(fn, "render modes 0 (6), 1 and 2 only");
    if (count >= (1ull << 32)) return invalid(fn, "too many gaussians (< 2^32 supported)");
    return aligned_ok(fn, "the record and quad buffers must be 16-byte aligned", {{d_quads, 16}, {d_records, 16}}) ? M2S_OK : M2S_E_INVALID;
}

// the kernel's arguments: the uniforms of GaussiansPrepass::execute; M2S_E_INVALID for a singular model matrix
static m2s_status prepass_fill(const void* d_records, uint64_t count, const uint64_t* d_count, const m2s_prepass_params* p, void* d_quads,
                               float* d_depths, uint32_t* d_valid, PrepassArgs& a) {
    std::memset(&a, 0, sizeof(a));
    std::memcpy(a.V, p->world_to_view, 64); std::memcpy(a.P, p->view_to_clip, 64); std::memcpy(a.M, p->model_to_world, 64);
    double M[16], Mi[16];
    for (int k = 0; k < 16; ++k) M[k] = p->model_to_world[k];
    if (!invert4(M, Mi)) { set_error("m2s_prepass: model_to_world is singular"); return M2S_E_INVALID; }
    for (int c = 0; c < 4; ++c) for (int r = 0; r < 4; ++r) a.Nmat[c * 4 + r] = (float)Mi[r * 4 + c];   // transpose(inverse(M))
    {   // inverse(mat3(M)): rows of M's upper 3x3
        const double m00 = M[0], m01 = M[4], m02 = M[8], m10 = M[1], m11 = M[5], m12 = M[9], m20 = M[2], m21 = M[6], m22 = M[10];
        const double det = m00 * (m11 * m22 - m12 * m21) - m01 * (m10 * m22 - m12 * m20) + m02 * (m10 * m21 - m11 * m20);
        if (det == 0.0) { set_error("m2s_prepass: model_to_world has a singular rotation part"); return M2S_E_INVALID; }
        const double i = 1.0 / det;
        a.Ninv[0] = (float)((m11 * m22 - m12 * m21) * i); a.Ninv[3] = (float)((m02 * m21 - m01 * m22) * i); a.Ninv[6] = (float)((m01 * m12 - m02 * m11) * i);
        a.Ninv[1] = (float)((m12 * m20 - m10 * m22) * i); a.Ninv[4] = (float)((m00 * m22 - m02 * m20) * i); a.Ninv[7] = (float)((m02 * m10 - m00 * m12) * i);
        a.Ninv[2] = (float)((m10 * m21 - m11 * m20) * i); a.Ninv[5] = (float)((m01 * m20 - m00 * m21) * i); a.Ninv[8] = (float)((m00 * m11 - m01 * m10) * i);
    }
    const double l0 = M[0] * M[0] + M[1] * M[1] + M[2] * M[2] + M[3] * M[3], l1 = M[4] * M[4] + M[5] * M[5] + M[6] * M[6] + M[7] * M[7];
    a.mscale2[0] = (float)l0; a.mscale2[1] = (float)l0; a.mscale2[2] = (float)l1;   // (|M[0]|, |M[0]|, |M[1]|) squared — sic (:96)
    a.res[0] = p->resolution[0]; a.res[1] = p->resolution[1]; a.near_far[0] = p->near_far[0]; a.near_far[1] = p->near_far[1];
    ViewInput v;
    view_input(p->layout, v);   // checked by prepass_check
    a.std_dev = p->std_dev; a.render_mode = p->render_mode; a.layout = v.layout; a.fmt = v.fmt; a.ply_has_pbr = v.ply_has_pbr;
    a.count = count; a.d_count = (const unsigned long long*)d_count;
    a.records = (const unsigned char*)d_records; a.quads = (float4*)d_quads; a.depths = d_depths; a.valid = d_valid;
    return M2S_OK;
}

M2S_EXPORT m2s_status m2s_prepass_enqueue(m2s_ctx* ctx, const void* d_records, uint64_t count, const uint64_t* d_count,
                                          const m2s_prepass_params* p, void* d_quads, float* d_depths, uint32_t* d_valid, void* stream_) {
    m2s_status st = prepass_check(ctx, d_records, count, p, d_quads, d_depths, d_valid != nullptr);
    if (st != M2S_OK) return st;
    CUDA_TRY(cudaSetDevice(ctx->device));
    cudaStream_t stream = pick_stream(ctx, stream_);
    PrepassArgs a;
    st = prepass_fill(d_records, count, d_count, p, d_quads, d_depths, d_valid, a);
    if (st != M2S_OK) return st;
    CUDA_TRY(cudaMemsetAsync(d_valid, 0, sizeof(uint32_t), stream));
    CUDA_TRY(prepass_launch(a, stream));
    return M2S_OK;
}

static m2s_status prepass_depth_check(const m2s_ctx* ctx, const void* d_records, uint64_t count, const m2s_prepass_params* p,
                                      const float* d_mesh_depth, uint32_t depth_width, uint32_t depth_height, const void* d_quads,
                                      const float* d_depths, bool has_valid) {
    const char* fn = "m2s_prepass_mesh_depth";
    m2s_status st = prepass_check(ctx, d_records, count, p, d_quads, d_depths, has_valid);
    if (st != M2S_OK) return st;
    if (!d_mesh_depth || (reinterpret_cast<uintptr_t>(d_mesh_depth) & 3u)) return invalid(fn, "the depth map must be a non-NULL, 4-byte aligned device buffer");
    return sizes_ok(fn, "depth_width and depth_height", kSplatMaxSide, {depth_width, depth_height}) ? M2S_OK : M2S_E_INVALID;
}

M2S_EXPORT m2s_status m2s_prepass_mesh_depth_enqueue(m2s_ctx* ctx, const void* d_records, uint64_t count, const uint64_t* d_count,
                                                     const m2s_prepass_params* p, const float* d_mesh_depth, uint32_t depth_width,
                                                     uint32_t depth_height, void* d_quads, float* d_depths, uint32_t* d_valid, void* stream_) {
    m2s_status st = prepass_depth_check(ctx, d_records, count, p, d_mesh_depth, depth_width, depth_height, d_quads, d_depths, d_valid != nullptr);
    if (st != M2S_OK) return st;
    PrepassDepthArgs a;
    st = prepass_fill(d_records, count, d_count, p, d_quads, d_depths, d_valid, a.p);
    if (st != M2S_OK) return st;
    a.map = d_mesh_depth; a.width = depth_width; a.height = depth_height;
    CUDA_TRY(cudaSetDevice(ctx->device));
    cudaStream_t stream = pick_stream(ctx, stream_);
    CUDA_TRY(cudaMemsetAsync(d_valid, 0, sizeof(uint32_t), stream));
    CUDA_TRY(prepass_depth_launch(a, stream));
    return M2S_OK;
}

// The synchronous prepass forms: enqueue(d_valid) runs the enqueue form on the context's stream with the context's
// counter, then the counter is read back into *valid (may be NULL).
template <typename Enqueue>
static m2s_status prepass_sync(m2s_ctx* ctx, uint32_t* valid, Enqueue enqueue) {
    CUDA_TRY(cudaSetDevice(ctx->device));
    if (!ctx->d_prepass_valid) CUDA_TRY(cudaMalloc(&ctx->d_prepass_valid, sizeof(uint32_t)));
    m2s_status st = enqueue(ctx->d_prepass_valid);
    if (st != M2S_OK) return st;
    uint32_t v = 0;
    CUDA_TRY(cudaMemcpyAsync(&v, ctx->d_prepass_valid, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    if (valid) *valid = v;
    return M2S_OK;
}

M2S_EXPORT m2s_status m2s_prepass(m2s_ctx* ctx, const void* d_records, uint64_t count, const m2s_prepass_params* p, void* d_quads,
                                  float* d_depths, uint32_t* valid) {
    if (!ctx) { set_error("m2s_prepass: ctx is NULL"); return M2S_E_INVALID; }
    return prepass_sync(ctx, valid, [&](uint32_t* d_valid) {
        return m2s_prepass_enqueue(ctx, d_records, count, nullptr, p, d_quads, d_depths, d_valid, ctx->stream);
    });
}

M2S_EXPORT m2s_status m2s_prepass_mesh_depth(m2s_ctx* ctx, const void* d_records, uint64_t count, const m2s_prepass_params* p,
                                             const float* d_mesh_depth, uint32_t depth_width, uint32_t depth_height, void* d_quads,
                                             float* d_depths, uint32_t* valid) {
    m2s_status st = prepass_depth_check(ctx, d_records, count, p, d_mesh_depth, depth_width, depth_height, d_quads, d_depths, true);
    if (st != M2S_OK) return st;
    return prepass_sync(ctx, valid, [&](uint32_t* d_valid) {
        return m2s_prepass_mesh_depth_enqueue(ctx, d_records, count, nullptr, p, d_mesh_depth, depth_width, depth_height, d_quads, d_depths,
                                              d_valid, ctx->stream);
    });
}

// ---- the viewer's depth sort (SURVEY 8 f-5): RadixSortPass::execute = radixSortPrepass.glsl + glu::RadixSort + radixSortGather.glsl
M2S_EXPORT m2s_status m2s_depth_sort_enqueue(m2s_ctx* ctx, const void* d_quads, const float* d_depths, uint64_t count,
                                             const uint32_t* d_count, void* d_sorted_quads, uint32_t* d_order, uint32_t* d_draw,
                                             void* stream_) {
    const char* fn = "m2s_depth_sort";
    if (!ctx) return invalid(fn, "ctx is NULL");
    if (count && (!d_quads || !d_depths || !d_sorted_quads)) return invalid(fn, "NULL argument");
    if (!aligned_ok(fn, "the quad buffers must be 16-byte aligned", {{d_quads, 16}, {d_sorted_quads, 16}})) return M2S_E_INVALID;
    if (count >= kSortMaxCount) return invalid(fn, "too many quads (< 2^30 supported)");
    if (count == 0 && !d_draw) return M2S_OK;
    CUDA_TRY(cudaSetDevice(ctx->device));
    cudaStream_t stream = pick_stream(ctx, stream_);
    const SortLayout l = sort_layout(count);
    if (count) {
        const m2s_status st = grow(ctx, ctx->sort, l.total_bytes, stream);
        if (st != M2S_OK) return st;
    }
    SortArgs a;
    a.count = count;
    a.d_count = d_count;
    a.depth_bits = reinterpret_cast<const uint32_t*>(d_depths);
    a.quads = static_cast<const float4*>(d_quads);
    a.sorted = static_cast<float4*>(d_sorted_quads);
    a.scratch = static_cast<uint32_t*>(ctx->sort.p);
    // without a caller's order buffer the permutation goes to the second value buffer, free by the last pass
    a.order = d_order ? d_order : (count ? a.scratch + l.ctrl_words + 3 * l.buf_words : nullptr);
    a.draw = d_draw;
    CUDA_TRY(sort_launch(a, ctx->sm_count, stream));
    return M2S_OK;
}

M2S_EXPORT m2s_status m2s_depth_sort(m2s_ctx* ctx, const void* d_quads, const float* d_depths, uint64_t count, void* d_sorted_quads,
                                     uint32_t* d_order, uint32_t* d_draw) {
    m2s_status st = m2s_depth_sort_enqueue(ctx, d_quads, d_depths, count, nullptr, d_sorted_quads, d_order, d_draw, nullptr);
    if (st != M2S_OK) return st;
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return M2S_OK;
}

// Test aid (not part of m2s.h): the number of keys one tile of a sort pass holds.
M2S_EXPORT uint32_t m2s_debug_sort_tile(void) { return (uint32_t)kSortTile; }

// ---- the binned passes (splat draw, cube raster, mesh depth pre-pass): count -> size -> draw ----------------------
// The steps after the pass's own front step has filled `a`, all on `stream`: size the pass's scratch (scratch_bytes,
// its BinLayout), count the pairs, size the pair sort for the budget, then emit, sort and draw.
//   enqueue form (sync false): the budget is max_pairs; the pair total and the drawn prefix are copied to the device
//       words pairs and d_drawn (either may be NULL).
//   synchronous form (sync true): the pair total is read back once and is the budget, 2^30 or more is rejected with
//       the pass's message too_many; the stream is synchronised and the total stored in the host word *pairs (may be
//       NULL).
// Each pass has one function that checks its arguments, fills `a` and calls this; its two entry points call that
// function with the form's sync, budget and pair words.
template <typename Args>
static m2s_status bin_pass(m2s_ctx* ctx, BinScratch& s, size_t scratch_bytes, Args& a, cudaError_t (*count)(const Args&, cudaStream_t),
                           cudaError_t (*draw)(const Args&, int, cudaStream_t), cudaStream_t stream, bool sync, uint64_t max_pairs,
                           uint64_t* pairs, uint32_t* d_drawn, const char* too_many) {
    m2s_status st = grow(ctx, s.bins, scratch_bytes, stream);
    if (st != M2S_OK) return st;
    a.scratch = static_cast<unsigned char*>(s.bins.p);
    CUDA_TRY(count(a, stream));
    if (sync) {
        CUDA_TRY(cudaMemcpyAsync(ctx->h_total, a.scratch, sizeof(uint64_t), cudaMemcpyDeviceToHost, stream));
        CUDA_TRY(cudaStreamSynchronize(stream));
        max_pairs = *ctx->h_total;
        if (max_pairs >= kSplatMaxPairs) { set_error(too_many); return M2S_E_INVALID; }
    }
    if (max_pairs) {
        st = grow(ctx, s.pairs, sort_layout(max_pairs).total_bytes, stream);
        if (st != M2S_OK) return st;
    }
    a.max_pairs = max_pairs;
    a.pairs = static_cast<uint32_t*>(s.pairs.p);
    CUDA_TRY(draw(a, ctx->sm_count, stream));
    if (sync) {
        CUDA_TRY(cudaStreamSynchronize(stream));
        if (pairs) *pairs = max_pairs;
        return M2S_OK;
    }
    if (pairs) CUDA_TRY(cudaMemcpyAsync(pairs, a.scratch, sizeof(uint64_t), cudaMemcpyDeviceToDevice, stream));
    if (d_drawn) CUDA_TRY(cudaMemcpyAsync(d_drawn, a.scratch + 8, sizeof(uint32_t), cudaMemcpyDeviceToDevice, stream));
    return M2S_OK;
}

// ---- the viewer's splat draw (SURVEY 8 f-6): GaussianSplattingPass::execute + gaussianSplattingVS/PS.glsl ----------
// both forms of the splat draw: the argument checks, the arguments, then bin_pass
static m2s_status splat_pass(m2s_ctx* ctx, const void* d_quads, uint64_t count, const uint32_t* d_draw, const m2s_splat_params* p,
                             const m2s_gbuffer* g, void* stream, bool sync, uint64_t max_pairs, uint64_t* pairs, uint32_t* d_drawn) {
    const char* fn = "m2s_splat_draw";
    if (!ctx || !p || !g) return invalid(fn, "NULL argument");
    if (count && !d_quads) return invalid(fn, "NULL quads");
    if (!aligned_ok(fn, "the quad buffer must be 16-byte aligned", {{d_quads, 16}})) return M2S_E_INVALID;
    if (count >= kSplatMaxCount) return invalid(fn, "too many quads (< 2^30 supported)");
    if (!pair_budget_ok(fn, max_pairs) || !sizes_ok(fn, "width and height", kSplatMaxSide, {p->width, p->height})) return M2S_E_INVALID;
    if (p->render_mode > 6) return invalid(fn, "render modes 0..6 only");
    if (!g->position && !g->normal && !g->albedo && !g->depth && !g->metallic_roughness) return invalid(fn, "no targets");
    if (!aligned_ok(fn, "RGBA16F targets must be 8-byte aligned, RGBA8 targets 4-byte aligned",
                    {{g->position, 8}, {g->normal, 8}, {g->depth, 8}, {g->albedo, 4}, {g->metallic_roughness, 4}}))
        return M2S_E_INVALID;
    CUDA_TRY(cudaSetDevice(ctx->device));
    SplatArgs a;
    std::memset(&a, 0, sizeof(a));
    a.quads = static_cast<const float4*>(d_quads);
    a.count = count;
    a.d_draw = d_draw;
    a.width = p->width; a.height = p->height; a.mode = p->render_mode;
    a.position = g->position; a.normal = g->normal; a.albedo = g->albedo; a.depth = g->depth; a.metallic_roughness = g->metallic_roughness;
    return bin_pass(ctx, ctx->splat_bins, bin_layout(count, splat_tiles(p->width, p->height)).total_bytes, a, splat_count_launch,
                    splat_draw_launch, pick_stream(ctx, stream), sync, max_pairs, pairs, d_drawn,
                    "m2s_splat_draw: the quads need 2^30 or more (tile, quad) pairs");
}

M2S_EXPORT m2s_status m2s_splat_draw_enqueue(m2s_ctx* ctx, const void* d_sorted_quads, uint64_t count, const uint32_t* d_draw,
                                             const m2s_splat_params* p, const m2s_gbuffer* g, uint64_t max_pairs, uint64_t* d_pairs,
                                             uint32_t* d_drawn, void* stream_) {
    return splat_pass(ctx, d_sorted_quads, count, d_draw, p, g, stream_, false, max_pairs, d_pairs, d_drawn);
}

M2S_EXPORT m2s_status m2s_splat_draw(m2s_ctx* ctx, const void* d_sorted_quads, uint64_t count, const m2s_splat_params* p,
                                     const m2s_gbuffer* g, uint64_t* pairs) {
    return splat_pass(ctx, d_sorted_quads, count, nullptr, p, g, nullptr, true, 0, pairs, nullptr);
}

// ---- the viewer's shadow pass (SURVEY 8 f-7): GaussianShadowPass::execute + gaussianPointShadowMappingCS.glsl + the
// cube face draws.  The uniforms are built on the host in fp32 with GLM's own formulas (lookAt, perspective, length,
// inverse(mat3)), the oracle restates the same steps (oracle/m2s_light_oracle.c orc_light_uniforms).
static void glm_normalize3(float v[3]) {
    const float inv = 1.0f / std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    v[0] = v[0] * inv; v[1] = v[1] * inv; v[2] = v[2] * inv;
}
static void glm_cross(const float a[3], const float b[3], float r[3]) {
    r[0] = a[1] * b[2] - b[1] * a[2]; r[1] = a[2] * b[0] - b[2] * a[0]; r[2] = a[0] * b[1] - b[0] * a[1];
}

static void shadow_uniforms(const m2s_shadow_params* p, ShadowArgs& a) {
    static const float kDir[6][3] = {{1, 0, 0}, {-1, 0, 0}, {0, 1, 0}, {0, -1, 0}, {0, 0, 1}, {0, 0, -1}};
    static const float kUp[6][3] = {{0, -1, 0}, {0, -1, 0}, {0, 0, 1}, {0, 0, -1}, {0, -1, 0}, {0, -1, 0}};
    const float* e = p->light_position;
    for (int f = 0; f < 6; ++f) {   // GaussianShadowPass.cpp:91-108: glm::lookAt(light, light + dir, up)
        float fw[3] = {(e[0] + kDir[f][0]) - e[0], (e[1] + kDir[f][1]) - e[1], (e[2] + kDir[f][2]) - e[2]}, s[3], u[3];
        glm_normalize3(fw);
        glm_cross(fw, kUp[f], s);
        glm_normalize3(s);
        glm_cross(s, fw, u);
        float* V = a.V[f];
        std::memset(V, 0, 64);
        V[0] = s[0]; V[4] = s[1]; V[8] = s[2];
        V[1] = u[0]; V[5] = u[1]; V[9] = u[2];
        V[2] = -fw[0]; V[6] = -fw[1]; V[10] = -fw[2];
        V[12] = -(s[0] * e[0] + s[1] * e[1] + s[2] * e[2]);
        V[13] = -(u[0] * e[0] + u[1] * e[1] + u[2] * e[2]);
        V[14] = fw[0] * e[0] + fw[1] * e[1] + fw[2] * e[2];
        V[15] = 1.0f;
    }
    // glm::perspective(glm::radians(90.0f), 1.0f, near, far) (:85), RH_NO
    const float n = p->near_far[0], fa = p->near_far[1];
    const float th = std::tan((90.0f * 0.01745329251994329576923690768489f) / 2.0f);
    std::memset(a.P, 0, 64);
    a.P[0] = 1.0f / (1.0f * th); a.P[5] = 1.0f / th;
    a.P[10] = -(fa + n) / (fa - n); a.P[11] = -1.0f; a.P[14] = -(2.0f * fa * n) / (fa - n);
    std::memcpy(a.M, p->model_to_world, 64);
    const float* M = p->model_to_world;
    // inverse(mat3(M)) (gaussianPointShadowMappingCS.glsl:104-110), GLM's compute_inverse<3, 3>; m[c][r] = M[4c + r]
    auto m = [M](int c, int r) { return M[4 * c + r]; };
    const float ood = 1.0f / (m(0, 0) * (m(1, 1) * m(2, 2) - m(2, 1) * m(1, 2)) - m(1, 0) * (m(0, 1) * m(2, 2) - m(2, 1) * m(0, 2)) +
                              m(2, 0) * (m(0, 1) * m(1, 2) - m(1, 1) * m(0, 2)));
    float* R = a.Rinv;   // column-major 3 x 3
    R[0] = (m(1, 1) * m(2, 2) - m(2, 1) * m(1, 2)) * ood;
    R[3] = -(m(1, 0) * m(2, 2) - m(2, 0) * m(1, 2)) * ood;
    R[6] = (m(1, 0) * m(2, 1) - m(2, 0) * m(1, 1)) * ood;
    R[1] = -(m(0, 1) * m(2, 2) - m(2, 1) * m(0, 2)) * ood;
    R[4] = (m(0, 0) * m(2, 2) - m(2, 0) * m(0, 2)) * ood;
    R[7] = -(m(0, 0) * m(2, 1) - m(2, 0) * m(0, 1)) * ood;
    R[2] = (m(0, 1) * m(1, 2) - m(1, 1) * m(0, 2)) * ood;
    R[5] = -(m(0, 0) * m(1, 2) - m(1, 0) * m(0, 2)) * ood;
    R[8] = (m(0, 0) * m(1, 1) - m(1, 0) * m(0, 1)) * ood;
    // modelScale = (length(M[0]), length(M[0]), length(M[1])) (:97), GLM vec4 dot (x x + y y) + (z z + w w); squared
    const float l0 = std::sqrt((M[0] * M[0] + M[1] * M[1]) + (M[2] * M[2] + M[3] * M[3]));
    const float l1 = std::sqrt((M[4] * M[4] + M[5] * M[5]) + (M[6] * M[6] + M[7] * M[7]));
    a.mscale2[0] = l0 * l0; a.mscale2[1] = l0 * l0; a.mscale2[2] = l1 * l1;
    for (int k = 0; k < 3; ++k) a.light[k] = e[k];
    a.res[0] = p->resolution[0]; a.res[1] = p->resolution[1];
    a.near_far[0] = n; a.near_far[1] = fa;
    a.std_dev = p->std_dev;
    ViewInput v;
    view_input(p->layout, v);   // checked by shadow_pass
    a.layout = v.layout;
    a.fmt = v.fmt;
    a.size = p->size;
}

// both forms of the shadow pass: the argument checks, the uniforms, the light records (the context's when the caller
// passes none), the light prepass, then the cube raster (bin_pass)
static m2s_status shadow_pass(m2s_ctx* ctx, const void* d_records, uint64_t count, const uint64_t* d_count, const m2s_shadow_params* p,
                              float* d_cube, void* d_light_quads, void* stream_, bool sync, uint64_t max_pairs, uint64_t* pairs,
                              uint32_t* d_drawn) {
    const char* fn = "m2s_shadow_map";
    if (!ctx || !p || !d_cube) return invalid(fn, "NULL argument");
    if (count && !d_records) return invalid(fn, "NULL records");
    ViewInput v;
    if (!view_input(p->layout, v)) return invalid(fn, "layouts REF96, PACKED56, VIEW_PLY and VIEW_PLY_PBR only");
    if (!aligned_ok(fn, "the record and light-record buffers must be 16-byte aligned, the cube 4-byte aligned",
                    {{d_records, 16}, {d_light_quads, 16}, {d_cube, 4}}))
        return M2S_E_INVALID;
    if (count >= kShadowMaxCount) return invalid(fn, "too many gaussians (< 2^30 supported)");
    if (!pair_budget_ok(fn, max_pairs) || !sizes_ok(fn, "size", kShadowMaxSize, {p->size})) return M2S_E_INVALID;
    CUDA_TRY(cudaSetDevice(ctx->device));
    cudaStream_t stream = pick_stream(ctx, stream_);
    ShadowArgs a;
    std::memset(&a, 0, sizeof(a));
    shadow_uniforms(p, a);
    if (!d_light_quads && count) {
        const m2s_status st = grow(ctx, ctx->light_quads, count * kLightRecordBytes, stream);
        if (st != M2S_OK) return st;
        d_light_quads = ctx->light_quads.p;
    }
    a.records = static_cast<const unsigned char*>(d_records);
    a.count = count;
    a.d_count = reinterpret_cast<const unsigned long long*>(d_count);
    a.light_quads = static_cast<float4*>(d_light_quads);
    a.cube = d_cube;
    CUDA_TRY(light_prepass_launch(a, stream));
    return bin_pass(ctx, ctx->shadow_bins, bin_layout(count, shadow_tiles(p->size)).total_bytes, a, shadow_count_launch, shadow_draw_launch,
                    stream, sync, max_pairs, pairs, d_drawn, "m2s_shadow_map: the records need 2^30 or more (tile, record) pairs");
}

M2S_EXPORT m2s_status m2s_shadow_map_enqueue(m2s_ctx* ctx, const void* d_records, uint64_t count, const uint64_t* d_count,
                                             const m2s_shadow_params* p, float* d_cube, void* d_light_quads, uint64_t max_pairs,
                                             uint64_t* d_pairs, uint32_t* d_drawn, void* stream_) {
    return shadow_pass(ctx, d_records, count, d_count, p, d_cube, d_light_quads, stream_, false, max_pairs, d_pairs, d_drawn);
}

M2S_EXPORT m2s_status m2s_shadow_map(m2s_ctx* ctx, const void* d_records, uint64_t count, const m2s_shadow_params* p, float* d_cube,
                                     void* d_light_quads, uint64_t* pairs) {
    return shadow_pass(ctx, d_records, count, nullptr, p, d_cube, d_light_quads, nullptr, true, 0, pairs, nullptr);
}

// ---- the viewer's deferred lighting (SURVEY 8 f-8): GaussianRelightingPass::execute + gaussianSplattingDeferredPS.glsl
M2S_EXPORT m2s_status m2s_deferred_light_enqueue(m2s_ctx* ctx, const m2s_gbuffer* g, const float* d_cube, const m2s_light_params* p,
                                                 uint8_t* d_image, void* stream_) {
    const char* fn = "m2s_deferred_light";
    if (!ctx || !g || !p || !d_image) return invalid(fn, "NULL argument");
    if (!sizes_ok(fn, "width and height", kSplatMaxSide, {p->width, p->height})) return M2S_E_INVALID;
    if (p->render_mode > 6) return invalid(fn, "render modes 0..6 only");
    const bool lit = p->render_mode == 6;
    if (!g->albedo || ((p->render_mode == 5 || lit) && !g->metallic_roughness) || (lit && (!g->position || !g->normal || !d_cube)))
        return invalid(fn, "NULL target or cube the render mode needs");
    if ((lit && !sizes_ok(fn, "shadow_size", kShadowMaxSize, {p->shadow_size})) ||
        !aligned_ok(fn, "RGBA16F targets must be 8-byte aligned, RGBA8 targets, the image and the cube 4-byte aligned",
                    {{g->position, 8}, {g->normal, 8}, {g->albedo, 4}, {g->metallic_roughness, 4}, {d_image, 4}, {d_cube, 4}}))
        return M2S_E_INVALID;
    CUDA_TRY(cudaSetDevice(ctx->device));
    LightArgs a;
    std::memset(&a, 0, sizeof(a));
    a.position = g->position; a.normal = g->normal; a.albedo = g->albedo; a.metallic_roughness = g->metallic_roughness;
    a.cube = d_cube;
    a.width = p->width; a.height = p->height; a.mode = p->render_mode; a.shadow_size = p->shadow_size;
    for (int k = 0; k < 3; ++k) { a.light[k] = p->light_position[k]; a.light_color[k] = p->light_color[k]; a.cam[k] = p->cam_pos[k]; }
    a.light_intensity = p->light_intensity; a.far_plane = p->far_plane;
    a.image = d_image;
    CUDA_TRY(deferred_light_launch(a, pick_stream(ctx, stream_)));
    return M2S_OK;
}

M2S_EXPORT m2s_status m2s_deferred_light(m2s_ctx* ctx, const m2s_gbuffer* g, const float* d_cube, const m2s_light_params* p, uint8_t* d_image) {
    m2s_status st = m2s_deferred_light_enqueue(ctx, g, d_cube, p, d_image, nullptr);
    if (st != M2S_OK) return st;
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return M2S_OK;
}

// ---- the viewer's mesh depth pre-pass (SURVEY 8 f-9): DepthPrepass::execute + depthPrepassVS/PS.glsl ----------------
// u_viewToClip * u_worldToView * u_modelToWorld as GLM evaluates it: (P V) M, each product GLM's mat4 * mat4 in fp32,
// r[c][row] = ((a[0][row] b[c][0] + a[1][row] b[c][1]) + a[2][row] b[c][2]) + a[3][row] b[c][3]
static void glm_mat4_mul(const float* a, const float* b, float* r) {
    for (int c = 0; c < 4; ++c)
        for (int row = 0; row < 4; ++row)
            r[c * 4 + row] = ((a[row] * b[c * 4] + a[4 + row] * b[c * 4 + 1]) + a[8 + row] * b[c * 4 + 2]) + a[12 + row] * b[c * 4 + 3];
}

// both forms of the mesh depth pre-pass: the argument checks, the arguments, then bin_pass
static m2s_status mesh_depth_pass(m2s_ctx* ctx, const m2s_dscene* scene, const m2s_mesh_depth_params* p, float* d_depth, void* stream,
                                  bool sync, uint64_t max_pairs, uint64_t* pairs, uint32_t* d_drawn) {
    const char* fn = "m2s_mesh_depth";
    if (!ctx || !scene || !p || !d_depth) return invalid(fn, "NULL argument");
    if (!aligned_ok(fn, "the depth map must be 4-byte aligned", {{d_depth, 4}}) ||
        !sizes_ok(fn, "width and height", kSplatMaxSide, {p->width, p->height}))
        return M2S_E_INVALID;
    if (scene->ntri >= kDepthMaxTris) return invalid(fn, "too many triangles (< 2^29 supported)");
    if (!pair_budget_ok(fn, max_pairs)) return M2S_E_INVALID;
    CUDA_TRY(cudaSetDevice(ctx->device));
    DepthArgs a;
    std::memset(&a, 0, sizeof(a));
    float pv[16];
    glm_mat4_mul(p->view_to_clip, p->world_to_view, pv);
    glm_mat4_mul(pv, p->model_to_world, a.pvm);
    a.tris = scene->d_tris;
    a.ntri = scene->ntri;
    a.ranges = scene->d_ranges;
    a.nranges = scene->nranges;
    a.prims = scene->d_prims;
    a.width = p->width;
    a.height = p->height;
    a.depth = d_depth;
    return bin_pass(ctx, ctx->depth_bins, bin_layout(a.ntri, splat_tiles(a.width, a.height)).total_bytes, a, depth_count_launch,
                    depth_draw_launch, pick_stream(ctx, stream), sync, max_pairs, pairs, d_drawn,
                    "m2s_mesh_depth: the triangles need 2^30 or more (tile, triangle) pairs");
}

M2S_EXPORT m2s_status m2s_mesh_depth_enqueue(m2s_ctx* ctx, const m2s_dscene* scene, const m2s_mesh_depth_params* p, float* d_depth,
                                             uint64_t max_pairs, uint64_t* d_pairs, uint32_t* d_drawn, void* stream_) {
    return mesh_depth_pass(ctx, scene, p, d_depth, stream_, false, max_pairs, d_pairs, d_drawn);
}

M2S_EXPORT m2s_status m2s_mesh_depth(m2s_ctx* ctx, const m2s_dscene* scene, const m2s_mesh_depth_params* p, float* d_depth, uint64_t* pairs) {
    return mesh_depth_pass(ctx, scene, p, d_depth, nullptr, true, 0, pairs, nullptr);
}
