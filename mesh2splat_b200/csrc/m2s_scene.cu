// m2s_scene.cu — C-ABI implementation (include/m2s.h): the device scene.  Eager and lazy upload, texture row groups and
// their mip rows, the v-range reduction that decides which rows a triangle range samples, and the shard upload.
#include "m2s_ctx.cuh"
#include "m2s_plane.cuh"

using namespace m2s;

namespace {

// ---- mip chain: 2x2 box, round half up (matches oracle orc_mip_down; GL_TEXTURE_MAX_LEVEL 4, glUtils.cpp:313) ----------
__device__ __forceinline__ uint32_t box4(uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    uint32_t o = 0;
#pragma unroll
    for (int s = 0; s < 32; s += 8) {
        const uint32_t sum = ((a >> s) & 0xff) + ((b >> s) & 0xff) + ((c >> s) & 0xff) + ((d >> s) & 0xff);
        o |= ((sum + 2) >> 2) << s;
    }
    return o;
}
// ALL levels of the 16-row groups [g0, g0 + gridDim.y) of one texture in one launch: a CTA takes 64 columns x 16 rows of
// level 0 and produces 32x8, 16x4, 8x2 and 4x1 texels of levels 1..4 (level l row j needs level l-1 rows 2j, 2j+1
// clamped to the last row: a 16-row group, and a 64-column tile, is closed under the filter).
__global__ void __launch_bounds__(256) mip_groups_kernel(uint32_t* __restrict__ arena, const DTexture t, uint32_t g0) {
    __shared__ uint32_t lv[3][8][32];  // levels 1..3 of this tile
    const uint32_t gx = blockIdx.x, g = g0 + blockIdx.y, tid = threadIdx.x;
    uint32_t cols = 32, rows = 8;
#pragma unroll
    for (uint32_t l = 1; l <= 4; ++l) {
        if (l < t.nlevels && tid < cols * rows) {
            const uint32_t lx = tid % cols, ly = tid / cols;
            const uint32_t x = gx * cols + lx, y = g * rows + ly;
            const uint32_t dw = t.w[l], dh = t.h[l], sw = t.w[l - 1], sh = t.h[l - 1];
            if (x < dw && y < dh) {
                const uint32_t x0 = min(2 * x, sw - 1), x1 = min(2 * x + 1, sw - 1), y0 = min(2 * y, sh - 1), y1 = min(2 * y + 1, sh - 1);
                uint32_t a, b, c, d;
                if (l == 1) {
                    const uint32_t* src = arena + t.off[0];
                    a = src[(size_t)y0 * sw + x0]; b = src[(size_t)y0 * sw + x1]; c = src[(size_t)y1 * sw + x0]; d = src[(size_t)y1 * sw + x1];
                } else {  // the source texels are this tile's own texels of the level above
                    const uint32_t bx = gx * cols * 2, by = g * rows * 2;
                    a = lv[l - 2][y0 - by][x0 - bx]; b = lv[l - 2][y0 - by][x1 - bx]; c = lv[l - 2][y1 - by][x0 - bx]; d = lv[l - 2][y1 - by][x1 - bx];
                }
                const uint32_t o = box4(a, b, c, d);
                arena[t.off[l] + (size_t)y * dw + x] = o;
                if (l < 4) lv[l - 1][ly][lx] = o;
            }
        }
        __syncthreads();
        cols >>= 1; rows >>= 1;
    }
}

// ---- the 64-byte position/uv stream of the PACKED56 raster pass (m2s_dscene::d_tris_slim) -----------------------------------
// One thread per output float4 k of triangle t: k < 3 is {P_k, u_k}, k = 3 is {v0, v1, v2, 0}; the values are copied, not computed.
// The thread of k = 3 also bounds the density at which the triangle's candidate box is small (small_box_density); the
// scene's minimum goes to *r_small (float bits, atomicMin: the bounds are >= 0), m2s_dscene::r_small_max.
__global__ void __launch_bounds__(256) slim_tris_kernel(const float4* __restrict__ tris, float4* __restrict__ slim, uint64_t n4,
                                                        const DRange* __restrict__ ranges, uint32_t nranges,
                                                        const DPrim* __restrict__ prims, uint32_t* __restrict__ r_small) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const float4* q = tris + (i >> 2) * 9;
    const uint32_t k = (uint32_t)i & 3u;
    float r = INFINITY;
    if (i < n4) {
        float4 o;
        if (k < 3) {
            const float4 p = __ldg(q + 3 * k), uv = __ldg(q + 3 * k + 2);
            o = make_float4(p.x, p.y, p.z, uv.z);
        } else {
            o = make_float4(__ldg(q + 2).w, __ldg(q + 5).w, __ldg(q + 8).w, 0.0f);
            const uint32_t t = (uint32_t)(i >> 2);
            int lo = 0, hi = (int)nranges - 1, found = -1;   // the set-up's triangle -> primitive search
            while (lo <= hi) {
                const int mid = (lo + hi) >> 1;
                const DRange rg = ranges[mid];
                if (t < rg.first) hi = mid - 1;
                else if (t >= rg.end) lo = mid + 1;
                else { found = (int)rg.prim; break; }
            }
            if (found >= 0) {
                f3 P[3], e1, n;
                float ou[3], ov[3];
#pragma unroll
                for (int v = 0; v < 3; ++v) { const float4 p = __ldg(q + 3 * v); P[v] = {p.x, p.y, p.z}; }
                ortho_uv(P, prims[found], e1, n, ou, ov);
                const float eu = fmaxf(ou[0], fmaxf(ou[1], ou[2])) - fminf(ou[0], fminf(ou[1], ou[2]));
                const float ev = fmaxf(ov[0], fmaxf(ov[1], ov[2])) - fminf(ov[0], fminf(ov[1], ov[2]));
                r = small_box_density(eu, ev);
            }
        }
        slim[i] = o;
    }
    const uint32_t m = __reduce_min_sync(0xffffffffu, __float_as_uint(r));
    if ((threadIdx.x & 31u) == 0 && m != __float_as_uint(INFINITY)) atomicMin(r_small, m);
}

// ---- v-range of a triangle range per texture (host pipeline: which texture rows must be uploaded before these triangles
// can be shaded).  minmax: [ntex] sortable-int minima | [ntex] maxima | 1 flag (non-finite or absurd v seen). -----------
__device__ __forceinline__ int float_key(float f) { const int i = __float_as_int(f); return i ^ ((i >> 31) & 0x7fffffff); }
__global__ void __launch_bounds__(256) vrange_kernel(const float4* __restrict__ tris, uint32_t first, uint32_t count,
                                                     const DRange* __restrict__ ranges, uint32_t nranges, const DPrim* __restrict__ prims,
                                                     uint32_t ntex, int* __restrict__ minmax) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    int prim = -1;
    float vmin = 3.0e38f, vmax = -3.0e38f;
    bool bad = false;
    if (i < count) {
        const uint32_t t = first + i;
        int lo = 0, hi = (int)nranges - 1;
        while (lo <= hi) {
            const int mid = (lo + hi) >> 1;
            const DRange r = ranges[mid];
            if (t < r.first) hi = mid - 1;
            else if (t >= r.end) lo = mid + 1;
            else { prim = (int)r.prim; break; }
        }
        if (prim >= 0) {
            const float v0 = __ldg(&tris[(size_t)t * 9 + 2]).w, v1 = __ldg(&tris[(size_t)t * 9 + 5]).w, v2 = __ldg(&tris[(size_t)t * 9 + 8]).w;
            vmin = fminf(v0, fminf(v1, v2)); vmax = fmaxf(v0, fmaxf(v1, v2));
            bad = !(fabsf(v0) <= 1e30f) || !(fabsf(v1) <= 1e30f) || !(fabsf(v2) <= 1e30f);
        }
    }
    const unsigned full = 0xffffffffu;
    if (__any_sync(full, bad) && lane == 0) atomicOr(minmax + 2 * ntex, 1);
    const int p0 = __shfl_sync(full, prim, 0);
    if (__all_sync(full, prim == p0)) {  // the usual case: the whole warp is inside one primitive
        if (p0 < 0) return;
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            vmin = fminf(vmin, __shfl_xor_sync(full, vmin, d));
            vmax = fmaxf(vmax, __shfl_xor_sync(full, vmax, d));
        }
        if (lane != 0) return;
    } else if (prim < 0) return;
    for (int m = 0; m < 3; ++m) {
        const int ti = prims[prim].tex[m];
        if (ti >= 0 && (uint32_t)ti < ntex) {
            atomicMin(minmax + ti, float_key(vmin));
            atomicMax(minmax + ntex + ti, float_key(vmax));
        }
    }
}

// The v-ranges of one chunk -> mapped pinned host memory, then a tag the host polls; the device copy is re-armed for its
// next use (min <- 0x7f7f7f7f, max <- 0x80808080, flag <- 0).  No copy engine: the download engine is busy with records,
// an 8-byte copy queued behind them reached the host 100-200 us late.
__global__ void vrange_publish_kernel(int* __restrict__ minmax, uint32_t ntex, volatile int* __restrict__ host, unsigned long long* host_tag,
                                      unsigned long long tag) {
    const uint32_t n = 2 * ntex + 1;
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        host[i] = minmax[i];
        minmax[i] = i < ntex ? 0x7f7f7f7f : (i < 2 * ntex ? (int)0x80808080 : 0);
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence_system();
        *reinterpret_cast<volatile unsigned long long*>(host_tag) = tag;
    }
}

}  // namespace

// levels 1.. of the 16-row groups [g0, g1) of one texture (level 0 must be resident), one launch
cudaError_t m2s::mip_groups_launch(uint32_t* arena, const DTexture& t, uint32_t g0, uint32_t g1, cudaStream_t stream) {
    if (t.nlevels <= 1 || g1 <= g0) return cudaSuccess;
    dim3 grd((t.w[0] + 63) / 64, g1 - g0);
    mip_groups_kernel<<<grd, 256, 0, stream>>>(arena, t, g0);
    return cudaGetLastError();
}

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
m2s_status m2s::upload_texture_groups(m2s_dscene* d, cudaStream_t stream, uint32_t t, uint32_t g0, uint32_t g1, std::vector<MipRun>* deferred) {
    const DTexture& dt = d->h_texs[t];
    const uint32_t H = dt.h[0], W = dt.w[0];
    const uint32_t r0 = g0 * kTexGroupRows, r1 = std::min<uint32_t>(H, g1 * kTexGroupRows);
    if (r0 >= r1) return M2S_OK;
    CUDA_TRY(cudaMemcpyAsync(d->d_arena + dt.off[0] + (size_t)r0 * W, d->h_rgba[t] + (size_t)r0 * W * 4, (size_t)(r1 - r0) * W * 4,
                             cudaMemcpyHostToDevice, stream));
    // level-l row j needs level-(l-1) rows 2j, 2j+1: inside the same 16-row group — all levels in one launch; inside the
    // host pipeline the launch is left to the caller (on the compute stream, behind an event: no kernel on the copy stream)
    const uint32_t ge = std::min<uint32_t>(g1, (H + kTexGroupRows - 1) / kTexGroupRows);
    if (deferred) deferred->push_back({t, g0, ge});
    else CUDA_TRY(mip_groups_launch(d->d_arena, dt, g0, ge, stream));
    for (uint32_t g = g0; g < g1 && g < d->present[t].size(); ++g) d->present[t][g] = 1;
    d->h2d_bytes += (uint64_t)(r1 - r0) * W * 4;
    return M2S_OK;
}

m2s_status m2s::vrange_enqueue(m2s_ctx* ctx, m2s_dscene* d, cudaStream_t stream, uint64_t lo, uint64_t hi, int slot) {
    const uint32_t nt = d->ntex;
    if (!nt) return M2S_OK;
    HostPipeline& hp = ctx->pipeline;
    if (hp.vr_ntex != nt) {  // (re)size and arm every slot: the armed layout (min block | max block | flag) depends on the texture count
        for (auto& v : hp.vr) {
            if (v.d_minmax) { cudaFree(v.d_minmax); v.d_minmax = nullptr; }
            if (v.h_minmax) { cudaFreeHost(v.h_minmax); v.h_minmax = nullptr; }
        }
        hp.vr_ntex = 0;
        for (auto& v : hp.vr) {
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
        hp.vr_ntex = nt;
    }
    VRangeSlot& v = hp.vr[slot];
    // min <- 0x7f7f7f7f (above every finite float's key), max <- 0x80808080 (below), flag <- 0
    // d_minmax is armed (at allocation, then by every publish kernel); a conversion that failed in between re-arms it
    if (hp.vr_dirty) {
        for (auto& w : hp.vr) {
            CUDA_TRY(cudaMemsetAsync(w.d_minmax, 0x7f, nt * sizeof(int), stream));
            CUDA_TRY(cudaMemsetAsync(w.d_minmax + nt, 0x80, nt * sizeof(int), stream));
            CUDA_TRY(cudaMemsetAsync(w.d_minmax + 2 * nt, 0, sizeof(int), stream));
        }
        hp.vr_dirty = false;
    }
    if (hi > lo) {
        vrange_kernel<<<(uint32_t)(hi - lo + 255) / 256, 256, 0, stream>>>(d->d_tris, (uint32_t)lo, (uint32_t)(hi - lo), d->d_ranges,
                                                                        d->nranges, d->d_prims, nt, v.d_minmax);
        CUDA_TRY(cudaGetLastError());
    }
    v.tag = ++hp.host_seq;
    vrange_publish_kernel<<<1, 128, 0, stream>>>(v.d_minmax, nt, v.h_minmax_dev, v.h_tag_dev, v.tag);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaEventRecord(v.ev, stream));
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
    // a scene uploaded whole gets the 64-byte stream its PACKED56 conversions stage (+64 B per triangle), built here once
    // behind the copies, and the density up to which every candidate box is small (r_small_max, read back once: it
    // decides per launch whether a conversion can end in the raster kernel); a partial or lazy upload would have to build
    // the stream per chunk and keeps the 144-byte route
    uint32_t* d_r_small = nullptr;
    if (sc->triangle_count && tri_offset == 0 && first_tris >= sc->triangle_count && !lazy_tex) {
        UP_TRY(dalloc((void**)&d->d_tris_slim, sc->triangle_count * (size_t)kSlimTriBytes));
        UP_TRY(dalloc((void**)&d_r_small, sizeof(uint32_t)));
        UP_TRY(cudaMemsetAsync(d_r_small, 0x7f, sizeof(uint32_t), ctx->stream));   // 3.4e38: no bound yet
        const uint64_t n4 = sc->triangle_count * 4;
        slim_tris_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, ctx->stream>>>(d->d_tris, d->d_tris_slim, n4, d->d_ranges,
                                                                                d->nranges, d->d_prims, d_r_small);
        UP_TRY(cudaGetLastError());
        UP_TRY(cudaMemcpyAsync(&d->r_small_max, d_r_small, sizeof(float), cudaMemcpyDeviceToHost, ctx->stream));
    }
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
            m2s_status st = upload_texture_groups(d, ctx->stream, t, 0, ngroups);
            if (st != M2S_OK) return fail(st);
        }
    }
    UP_TRY(dalloc((void**)&d->d_texs, d->h_texs.size() * sizeof(DTexture)));
    if (!d->h_texs.empty())
        UP_TRY(cudaMemcpyAsync(d->d_texs, d->h_texs.data(), d->h_texs.size() * sizeof(DTexture), cudaMemcpyHostToDevice, ctx->stream));
    if (sync || d_r_small) UP_TRY(cudaStreamSynchronize(ctx->stream));   // r_small_max has landed
#undef UP_TRY
    *out = d;
    return M2S_OK;
}

M2S_EXPORT m2s_status m2s_scene_upload(m2s_ctx* ctx, const m2s_scene* sc, m2s_dscene** out) {
    return scene_upload_impl(ctx, sc, out, UINT64_MAX, true);
}

M2S_EXPORT uint64_t m2s_scene_h2d_bytes(const m2s_dscene* s) { return s ? s->h2d_bytes : 0; }

// Test aid (not part of m2s.h): the scene's r_small_max (m2s_dscene); 0 when it has no slim triangle stream
M2S_EXPORT float m2s_debug_scene_r_small_max(const m2s_dscene* s) { return s ? s->r_small_max : 0.0f; }

// Test aid (not part of m2s.h): copies the scene's 64-byte position/uv stream (4 float4 per triangle) to host memory `dst`;
// M2S_E_INVALID when the scene has none (partial and lazy uploads)
M2S_EXPORT m2s_status m2s_debug_scene_slim_tris(m2s_ctx* ctx, const m2s_dscene* s, void* dst) {
    if (!ctx || !s || !dst) { set_error("m2s_debug_scene_slim_tris: NULL argument"); return M2S_E_INVALID; }
    if (!s->d_tris_slim) { set_error("m2s_debug_scene_slim_tris: the scene has no slim triangle stream"); return M2S_E_INVALID; }
    CUDA_TRY(cudaSetDevice(ctx->device));
    CUDA_TRY(cudaMemcpyAsync(dst, s->d_tris_slim, s->ntri * (size_t)kSlimTriBytes, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return M2S_OK;
}

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
    st = vrange_enqueue(ctx, ds, ctx->stream, r.first, r.first + r.count, 0);
    if (st == M2S_OK) st = upload_groups_from_vrange(ctx, ds, ctx->stream, 0, [] { return M2S_OK; });
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (st == M2S_OK && e != cudaSuccess) { set_error(std::string("m2s_scene_upload_range: ") + cudaGetErrorString(e)); st = M2S_E_CUDA; }
    if (st != M2S_OK) { m2s_scene_free(ctx, ds); return st; }
    *out = ds;
    return M2S_OK;
}
