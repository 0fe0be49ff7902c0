// m2s_scene.cu — C-ABI implementation (include/m2s.h): the device scene.  Eager and lazy upload, texture row groups and
// their mip rows, the v-range reduction that decides which rows a triangle range samples, and the shard upload.
#include "m2s_ctx.cuh"

using namespace m2s;

// ---- inputs ---------------------------------------------------------------------------------
M2S_EXPORT m2s_status m2s_compute_bboxes(const float* tris, m2s_primitive* prims, uint32_t nprim, int cumulative) {
    if ((!tris && nprim) || (!prims && nprim)) { set_error("m2s_compute_bboxes: NULL input"); return M2S_E_INVALID; }
    // SceneManager.cpp:476-477,514-520,527 — minBB/maxBB live outside the mesh loop
    float mn[3] = {3.402823466e+38f, 3.402823466e+38f, 3.402823466e+38f};
    float mx[3] = {-3.402823466e+38f, -3.402823466e+38f, -3.402823466e+38f};
    for (uint32_t p = 0; p < nprim; ++p) {
        if (!cumulative)
            for (int c = 0; c < 3; ++c) { mn[c] = 3.402823466e+38f; mx[c] = -3.402823466e+38f; }
        const uint64_t a = prims[p].first_triangle, b = a + prims[p].triangle_count;
        for (uint64_t t = a; t < b; ++t)
            for (int k = 0; k < 3; ++k)
                for (int c = 0; c < 3; ++c) {
                    const float v = tris[t * M2S_FLOATS_PER_TRIANGLE + M2S_FLOATS_PER_VERTEX * k + c];
                    mn[c] = std::min(mn[c], v);
                    mx[c] = std::max(mx[c], v);
                }
        for (int c = 0; c < 3; ++c) { prims[p].bbox_min[c] = mn[c]; prims[p].bbox_max[c] = mx[c]; }
    }
    return M2S_OK;
}

static uint32_t mip_levels(uint32_t w, uint32_t h) {
    uint32_t m = std::max(w, h), q = 0;
    while ((m >> (q + 1)) != 0) ++q;
    return std::min<uint32_t>(q, M2S_MAX_MIP_LEVEL) + 1;
}

M2S_EXPORT void m2s_scene_free(m2s_ctx* ctx, m2s_dscene* s) {
    if (!s) return;
    if (ctx) {
        cudaSetDevice(ctx->device);
        for (void* p : s->allocs) cudaFreeAsync(p, ctx->stream);
    }
    delete s;
}

// one contiguous H2D copy, then the rows of levels 1.. that they determine
m2s_status m2s::upload_texture_groups(m2s_ctx* ctx, m2s_dscene* d, uint32_t t, uint32_t g0, uint32_t g1, std::vector<MipRun>* deferred) {
    const DTexture& dt = d->h_texs[t];
    const uint32_t H = dt.h[0], W = dt.w[0];
    const uint32_t r0 = g0 * kTexGroupRows, r1 = std::min<uint32_t>(H, g1 * kTexGroupRows);
    if (r0 >= r1) return M2S_OK;
    CUDA_TRY(cudaMemcpyAsync(d->d_arena + dt.off[0] + (size_t)r0 * W, d->h_rgba[t] + (size_t)r0 * W * 4, (size_t)(r1 - r0) * W * 4,
                             cudaMemcpyHostToDevice, ctx->tex_up));
    // level-l row j needs level-(l-1) rows 2j, 2j+1: inside the same 16-row group — all levels in one launch; inside the
    // host pipeline the launch is left to the caller (on the compute stream, behind an event: no kernel on the copy stream)
    const uint32_t ge = std::min<uint32_t>(g1, (H + kTexGroupRows - 1) / kTexGroupRows);
    if (deferred) deferred->push_back({t, g0, ge});
    else CUDA_TRY(mip_groups_launch(d->d_arena, dt, g0, ge, ctx->tex_up));
    for (uint32_t g = g0; g < g1 && g < d->present[t].size(); ++g) d->present[t][g] = 1;
    d->h2d_bytes += (uint64_t)(r1 - r0) * W * 4;
    return M2S_OK;
}

m2s_status m2s::vrange_enqueue(m2s_ctx* ctx, m2s_dscene* d, uint64_t lo, uint64_t hi, int slot) {
    const uint32_t nt = d->ntex;
    if (!nt) return M2S_OK;
    if (ctx->vr_ntex != nt) {  // (re)size and arm every slot: the armed layout (min block | max block | flag) depends on the texture count
        for (auto& v : ctx->vr) {
            if (v.d_minmax) { cudaFree(v.d_minmax); v.d_minmax = nullptr; }
            if (v.h_minmax) { cudaFreeHost(v.h_minmax); v.h_minmax = nullptr; }
        }
        ctx->vr_ntex = 0;
        for (auto& v : ctx->vr) {
            const size_t nints = 2 * (size_t)nt + 1, tag_off = (nints * sizeof(int) + 7) & ~(size_t)7;
            CUDA_TRY(cudaMalloc(&v.d_minmax, nints * sizeof(int)));
            std::vector<int> arm(nints, 0);
            for (size_t i = 0; i < nt; ++i) { arm[i] = 0x7f7f7f7f; arm[nt + i] = (int)0x80808080; }
            CUDA_TRY(cudaMemcpy(v.d_minmax, arm.data(), nints * sizeof(int), cudaMemcpyHostToDevice));
            CUDA_TRY(cudaHostAlloc(&v.h_minmax, tag_off + 8, cudaHostAllocMapped));
            std::memset(v.h_minmax, 0, tag_off + 8);
            CUDA_TRY(cudaHostGetDevicePointer((void**)&v.h_minmax_dev, v.h_minmax, 0));
            v.h_tag = reinterpret_cast<unsigned long long*>(reinterpret_cast<unsigned char*>(v.h_minmax) + tag_off);
            v.h_tag_dev = reinterpret_cast<unsigned long long*>(reinterpret_cast<unsigned char*>(v.h_minmax_dev) + tag_off);
            if (!v.ev) CUDA_TRY(cudaEventCreateWithFlags(&v.ev, cudaEventDisableTiming));
        }
        ctx->vr_ntex = nt;
    }
    VRangeSlot& v = ctx->vr[slot];
    // min <- 0x7f7f7f7f (above every finite float's key), max <- 0x80808080 (below), flag <- 0
    // d_minmax is armed (at allocation, then by every publish kernel); a conversion that failed in between re-arms it
    if (ctx->vr_dirty) {
        for (auto& w : ctx->vr) {
            CUDA_TRY(cudaMemsetAsync(w.d_minmax, 0x7f, nt * sizeof(int), ctx->aux));
            CUDA_TRY(cudaMemsetAsync(w.d_minmax + nt, 0x80, nt * sizeof(int), ctx->aux));
            CUDA_TRY(cudaMemsetAsync(w.d_minmax + 2 * nt, 0, sizeof(int), ctx->aux));
        }
        ctx->vr_dirty = false;
    }
    if (hi > lo)
        CUDA_TRY(vrange_launch(d->d_tris, (uint32_t)lo, (uint32_t)(hi - lo), d->d_ranges, d->nranges, d->d_prims, nt, v.d_minmax, ctx->aux));
    v.tag = ++ctx->host_seq;
    CUDA_TRY(vrange_publish_launch(v.d_minmax, nt, v.h_minmax_dev, v.h_tag_dev, v.tag, ctx->aux));
    CUDA_TRY(cudaEventRecord(v.ev, ctx->aux));
    return M2S_OK;
}

m2s_status m2s::scene_upload_impl(m2s_ctx* ctx, const m2s_scene* sc, m2s_dscene** out, uint64_t first_tris, bool sync,
                                  uint64_t tri_offset, bool lazy_tex) {
    if (!ctx || !sc || !out) { set_error("m2s_scene_upload: NULL argument"); return M2S_E_INVALID; }
    *out = nullptr;
    if (sc->triangle_count && !sc->triangles) { set_error("m2s_scene_upload: triangles is NULL"); return M2S_E_INVALID; }
    if (sc->triangle_count >= (1ull << 32) - 64) { set_error("m2s_scene_upload: too many triangles (< 2^32 supported)"); return M2S_E_INVALID; }
    if ((sc->primitive_count && !sc->primitives) || (sc->texture_count && !sc->textures)) {
        set_error("m2s_scene_upload: primitive/texture table is NULL"); return M2S_E_INVALID;
    }
    // primitive ranges: inside the triangle list, pairwise disjoint
    std::vector<DRange> ranges;
    std::vector<DPrim> prims(sc->primitive_count);
    for (uint32_t p = 0; p < sc->primitive_count; ++p) {
        const m2s_primitive& src = sc->primitives[p];
        if (src.first_triangle + src.triangle_count > sc->triangle_count) {
            set_error("m2s_scene_upload: primitive range exceeds the triangle list"); return M2S_E_INVALID;
        }
        const int32_t ti[3] = {src.albedo_texture, src.normal_texture, src.metallic_roughness_texture};
        for (int m = 0; m < 3; ++m) {
            if (ti[m] >= (int32_t)sc->texture_count) { set_error("m2s_scene_upload: texture index out of range"); return M2S_E_INVALID; }
            prims[p].tex[m] = ti[m] < 0 ? -1 : ti[m];
        }
        for (int c = 0; c < 3; ++c) { prims[p].bmin[c] = src.bbox_min[c]; prims[p].bmax[c] = src.bbox_max[c]; }
        for (int c = 0; c < 4; ++c) prims[p].factor[c] = src.base_color_factor[c];
        prims[p].pad = 0;
        if (src.triangle_count)
            ranges.push_back({(uint32_t)src.first_triangle, (uint32_t)(src.first_triangle + src.triangle_count), p, 0});
    }
    std::sort(ranges.begin(), ranges.end(), [](const DRange& a, const DRange& b) { return a.first < b.first; });
    for (size_t i = 1; i < ranges.size(); ++i)
        if (ranges[i].first < ranges[i - 1].end) { set_error("m2s_scene_upload: primitive triangle ranges overlap"); return M2S_E_INVALID; }
    for (uint32_t t = 0; t < sc->texture_count; ++t)
        if (!sc->textures[t].rgba || !sc->textures[t].width || !sc->textures[t].height ||
            sc->textures[t].width > 32768 || sc->textures[t].height > 32768) {
            set_error("m2s_scene_upload: bad texture"); return M2S_E_INVALID;
        }

    CUDA_TRY(cudaSetDevice(ctx->device));
    m2s_dscene* d = new m2s_dscene();
    auto fail = [&](m2s_status st) { m2s_scene_free(ctx, d); return st; };
#define UP_TRY(expr)                                                                 \
    do {                                                                             \
        cudaError_t _e = (expr);                                                     \
        if (_e != cudaSuccess) {                                                     \
            set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));           \
            return fail(M2S_E_CUDA);                                                 \
        }                                                                            \
    } while (0)
    auto dalloc = [&](void** p, size_t bytes) -> cudaError_t {
        cudaError_t e = cudaMallocAsync(p, std::max<size_t>(bytes, 16), ctx->stream);
        if (e == cudaSuccess) d->allocs.push_back(*p);
        return e;
    };
    d->ntri = sc->triangle_count;
    UP_TRY(dalloc((void**)&d->d_tris, sc->triangle_count * (size_t)kTriBytes));
    if (sc->triangle_count && tri_offset < sc->triangle_count && first_tris)  // triangles [tri_offset, tri_offset + first_tris)
        UP_TRY(cudaMemcpyAsync(reinterpret_cast<unsigned char*>(d->d_tris) + tri_offset * (size_t)kTriBytes,
                               reinterpret_cast<const unsigned char*>(sc->triangles) + tri_offset * (size_t)kTriBytes,
                               std::min<uint64_t>(first_tris, sc->triangle_count - tri_offset) * (size_t)kTriBytes, cudaMemcpyHostToDevice, ctx->stream));
    if (sc->triangle_count && tri_offset < sc->triangle_count && first_tris)
        d->h2d_bytes += std::min<uint64_t>(first_tris, sc->triangle_count - tri_offset) * (uint64_t)kTriBytes;
    d->nranges = (uint32_t)ranges.size();
    UP_TRY(dalloc((void**)&d->d_ranges, ranges.size() * sizeof(DRange)));
    if (!ranges.empty())
        UP_TRY(cudaMemcpyAsync(d->d_ranges, ranges.data(), ranges.size() * sizeof(DRange), cudaMemcpyHostToDevice, ctx->stream));
    d->nprims = sc->primitive_count;
    UP_TRY(dalloc((void**)&d->d_prims, prims.size() * sizeof(DPrim)));
    if (!prims.empty())
        UP_TRY(cudaMemcpyAsync(d->d_prims, prims.data(), prims.size() * sizeof(DPrim), cudaMemcpyHostToDevice, ctx->stream));
    // textures: ONE arena for all mip chains (levels addressed by 32-bit texel offsets); levels 1..
    // are built on the GPU
    d->ntex = sc->texture_count;
    d->h_texs.resize(sc->texture_count);
    size_t arena_texels = 64;
    for (uint32_t t = 0; t < sc->texture_count; ++t) {
        DTexture& dt = d->h_texs[t];
        std::memset(&dt, 0, sizeof(dt));
        dt.nlevels = mip_levels(sc->textures[t].width, sc->textures[t].height);
        uint32_t w = sc->textures[t].width, h = sc->textures[t].height;
        for (uint32_t l = 0; l < (uint32_t)kMaxLevels; ++l) {
            if (l < dt.nlevels) {
                dt.w[l] = (uint16_t)w; dt.h[l] = (uint16_t)h;
                if (arena_texels + (size_t)w * h >= (1ull << 32)) { set_error("m2s_scene_upload: textures exceed the 16 GiB arena"); return fail(M2S_E_INVALID); }
                dt.off[l] = (uint32_t)arena_texels;
                arena_texels += (size_t)w * h;
                arena_texels = (arena_texels + 63) & ~(size_t)63;  // 256-byte aligned levels
                w = std::max(1u, w / 2); h = std::max(1u, h / 2);
            } else { dt.w[l] = dt.w[dt.nlevels - 1]; dt.h[l] = dt.h[dt.nlevels - 1]; dt.off[l] = dt.off[dt.nlevels - 1]; }
        }
    }
    UP_TRY(dalloc((void**)&d->d_arena, arena_texels * 4));
    d->h_rgba.resize(sc->texture_count);
    d->present.resize(sc->texture_count);
    for (uint32_t t = 0; t < sc->texture_count; ++t) {
        const uint32_t ngroups = (d->h_texs[t].h[0] + kTexGroupRows - 1) / kTexGroupRows;
        d->h_rgba[t] = sc->textures[t].rgba;
        d->present[t].assign(ngroups, 0);
        if (!lazy_tex) {
            m2s_status st = upload_texture_groups(ctx, d, t, 0, ngroups);
            if (st != M2S_OK) return fail(st);
        }
    }
    UP_TRY(dalloc((void**)&d->d_texs, d->h_texs.size() * sizeof(DTexture)));
    if (!d->h_texs.empty())
        UP_TRY(cudaMemcpyAsync(d->d_texs, d->h_texs.data(), d->h_texs.size() * sizeof(DTexture), cudaMemcpyHostToDevice, ctx->stream));
    if (sync) UP_TRY(cudaStreamSynchronize(ctx->stream));
#undef UP_TRY
    *out = d;
    return M2S_OK;
}

M2S_EXPORT m2s_status m2s_scene_upload(m2s_ctx* ctx, const m2s_scene* sc, m2s_dscene** out) {
    return scene_upload_impl(ctx, sc, out, UINT64_MAX, true);
}

M2S_EXPORT uint64_t m2s_scene_h2d_bytes(const m2s_dscene* s) { return s ? s->h2d_bytes : 0; }

M2S_EXPORT m2s_status m2s_scene_read_mip(m2s_ctx* ctx, const m2s_dscene* s, uint32_t texture, uint32_t level, uint8_t* dst,
                                         uint32_t* width, uint32_t* height) {
    if (!ctx || !s || !dst) { set_error("m2s_scene_read_mip: NULL argument"); return M2S_E_INVALID; }
    if (texture >= s->ntex || level >= s->h_texs[texture].nlevels) { set_error("m2s_scene_read_mip: out of range"); return M2S_E_INVALID; }
    const DTexture& t = s->h_texs[texture];
    CUDA_TRY(cudaSetDevice(ctx->device));
    CUDA_TRY(cudaMemcpyAsync(dst, s->d_arena + t.off[level], (size_t)t.w[level] * t.h[level] * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    if (width) *width = t.w[level];
    if (height) *height = t.h[level];
    return M2S_OK;
}

// One shard of a scene: the triangles [first, first + count) (at their global indices) and only the texture rows they
// can sample, only the maps `layout` consumes — what one rank of a multi-GPU conversion needs on its device.
M2S_EXPORT m2s_status m2s_scene_upload_range(m2s_ctx* ctx, const m2s_scene* sc, uint32_t layout, uint64_t first_triangle,
                                             uint64_t triangle_count, m2s_dscene** out) {
    if (!ctx || !sc || !out) { set_error("m2s_scene_upload_range: NULL argument"); return M2S_E_INVALID; }
    if (layout > M2S_LAYOUT_PLY_COMPRESSED) { set_error("m2s_scene_upload_range: unknown layout"); return M2S_E_INVALID; }
    CUDA_TRY(cudaSetDevice(ctx->device));
    SlimScene slim(sc, layout);
    const TriRange r = tri_range(first_triangle, triangle_count, sc->triangle_count);
    m2s_dscene* ds = nullptr;
    m2s_status st = scene_upload_impl(ctx, &slim.scene, &ds, r.count, false, r.first, true);
    if (st != M2S_OK) return st;
    st = vrange_enqueue(ctx, ds, r.first, r.first + r.count, 0);
    if (st == M2S_OK) st = upload_groups_from_vrange(ctx, ds, 0, [] { return cudaSuccess; });
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (st == M2S_OK && e != cudaSuccess) { set_error(std::string("m2s_scene_upload_range: ") + cudaGetErrorString(e)); st = M2S_E_CUDA; }
    if (st != M2S_OK) { m2s_scene_free(ctx, ds); return st; }
    *out = ds;
    return M2S_OK;
}
