// m2s_convert.cu — C-ABI implementation (include/m2s.h): the conversion.  Its launch plan, the enqueue and synchronous
// forms, the pipelined host-to-host conversion (m2s_convert_host), and the .ply outputs.
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>

#include "m2s_ctx.cuh"

using namespace m2s;

static unsigned long long* g_trace = nullptr;  // debugging aid for M2S_TRACE builds (scripts/trace_raster.py)
M2S_EXPORT void m2s_debug_set_trace(void* p) { g_trace = (unsigned long long*)p; }

// ---- the hot path -----------------------------------------------------------------------------
uint64_t m2s::effective_cap(const m2s_dscene* s, const m2s_params* p, uint64_t out_capacity) {
    uint64_t cap = p->max_gaussians;
    if (cap == 0) cap = (p->flags & M2S_FLAG_UNCAPPED) ? out_capacity : m2s_reference_capacity(p->resolution, s->nprims);
    return std::min(cap, out_capacity);
}

// more records were generated than the conversion could store
static m2s_status capacity_error(uint64_t total, uint64_t cap) {
    char buf[160];
    std::snprintf(buf, sizeof(buf), "m2s_convert: %llu gaussians generated, capacity %llu", (unsigned long long)total, (unsigned long long)cap);
    set_error(buf);
    return M2S_E_CAPACITY;
}

// The launch plan of one conversion: what the two kernels are launched with and which route the raster kernel takes.
// One function computes it for the launch and for m2s_debug_convert_plan, so the route a test reads is the route the
// kernel runs.  Every field is a u64 (the ctypes mirror is _abi.m2s_convert_plan).
struct ConvertPlan {
    uint64_t grid, raster_warps;      // raster CTAs, and their warps
    uint64_t unit_tris, n_units;      // work units of the triangle range
    uint64_t item_max, flush_frags;   // fragment work-item sizes
    uint64_t queue_cap;               // work-item queue slots
    uint64_t cap;                     // records stored (the effective cap)
    uint64_t multi_round;             // n_units > raster_warps: the warps take several units each
    uint64_t direct_ok;               // the raster kernel shades light units itself (PACKED56, multi-round, one GPU)
    uint64_t claim_late;              // ... and claims a warp's next unit once its current one is done (< 3 units per warp)
    uint64_t direct_max;              // M2S_DIRECT_MAX: the heaviest unit (small-triangle fragments) the direct path takes
};

static void convert_plan(const m2s_ctx* ctx, const m2s_dscene* s, const m2s_params* p, uint64_t out_capacity, uint32_t world,
                         ConvertPlan* pl) {
    const uint64_t count = tri_range(p->first_triangle, p->triangle_count, s->ntri).count;
    const int klayout = (int)p->layout;
    pl->cap = effective_cap(s, p, out_capacity);
    pl->grid = (uint64_t)ctx->sm_count * ctx->blocks_per_sm[klayout];
    pl->raster_warps = pl->grid * convert_warps_per_cta(klayout);
    // work-unit size: as large as 32 triangles, but small enough that every warp of the grid gets the
    // same number of units (a 70 k-triangle mesh is only ~1 unit of 32 per resident warp)
    const uint64_t warps = pl->raster_warps;
    const uint64_t rounds = std::max<uint64_t>(1, (count + warps * kUnitTris - 1) / (warps * kUnitTris));
    pl->unit_tris = std::min<uint64_t>(std::max<uint64_t>((count + warps * rounds - 1) / (warps * rounds), 1), kUnitTris);
    pl->n_units = (count + pl->unit_tris - 1) / pl->unit_tris;
    // work-item granularity: ~8 items per SM at the expected output (O(2 R^2) fragments) so that small conversions
    // still spread over the GPU, at most 2048 fragments; an oversized row block (<= 32 rows x R pixels) takes at most
    // kMaxSplit queue slots
    uint32_t item_max = (uint32_t)std::min<uint64_t>(kItemMaxFrags, (2ull * p->resolution * p->resolution) / ((uint64_t)ctx->sm_count * 8));
    item_max = std::max<uint32_t>({item_max, 64u, (32u * p->resolution + kMaxSplit - 1) / kMaxSplit});
    item_max = std::min<uint32_t>((item_max + 31u) & ~31u, kItemMaxFrags);
    pl->item_max = item_max;
    pl->flush_frags = std::max<uint32_t>(32u, item_max / 2);
    // item queue: a warp stops taking slots once it has seen the counter pass the cap, so live items cover disjoint
    // output ranges below it: per unit one item of small triangles and one end-of-unit item, cap/32 items closed by
    // 32 non-empty blocks, cap/flush closed by their fragment count, cap/item_max pieces of oversized blocks; plus
    // ONE reservation per raster warp that may straddle the cap (< 2 kMaxSplit + kStashItems slots).  The queue
    // cannot overflow.
    pl->queue_cap = std::min<uint64_t>(2 * pl->n_units + pl->cap / 32 + pl->cap / pl->flush_frags + pl->cap / pl->item_max +
                                       warps * (2ull * kMaxSplit + kStashItems) + 64, (1u << 24) - 1);
    pl->multi_round = pl->n_units > warps;
#ifndef M2S_EXP_NODIRECT
    pl->direct_ok = klayout == M2S_LAYOUT_PACKED56 && pl->multi_round && world <= 1;
#else
    pl->direct_ok = 0;
#endif
    // the late claim evens out the weights of the direct units when each warp gets only two of them; with more units
    // per warp they average out anyway and the claim's exposed atomic round trip is not worth it (DESIGN §4)
    pl->claim_late = pl->direct_ok && pl->n_units < 3 * warps;
    pl->direct_max = M2S_DIRECT_MAX;
}

// Test and tuning aid (not part of m2s.h): the plan m2s_convert would launch with for these arguments.  `plan` receives
// the fields of ConvertPlan in order.
M2S_EXPORT m2s_status m2s_debug_convert_plan(m2s_ctx* ctx, const m2s_dscene* s, const m2s_params* p, uint64_t out_capacity, uint64_t* plan) {
    if (!ctx || !s || !p || !plan) { set_error("m2s_debug_convert_plan: NULL argument"); return M2S_E_INVALID; }
    if (p->resolution < 1 || p->resolution > 4096 || p->layout > M2S_LAYOUT_PLY_COMPRESSED) { set_error("m2s_debug_convert_plan: bad params"); return M2S_E_INVALID; }
    ConvertPlan pl;
    convert_plan(ctx, s, p, out_capacity, 1u, &pl);
    std::memcpy(plan, &pl, sizeof(pl));
    return M2S_OK;
}

m2s_status m2s::convert_enqueue_impl(m2s_ctx* ctx, const m2s_dscene* s, const m2s_params* p, void* d_out, uint64_t out_capacity,
                                     uint64_t* d_keys, uint64_t* d_total, void* stream_, const m2s_peers* peers,
                                     const unsigned long long* prev_totals, uint32_t nprev,
                                     unsigned long long* host_total, unsigned long long host_tag, cudaEvent_t mid) {
    if (!ctx || !s || !p) { set_error("m2s_convert: NULL argument"); return M2S_E_INVALID; }
    if (p->resolution < 1 || p->resolution > 4096) { set_error("m2s_convert: resolution must be in 1..4096"); return M2S_E_INVALID; }
    if (p->layout > M2S_LAYOUT_PLY_COMPRESSED) { set_error("m2s_convert: unknown layout"); return M2S_E_INVALID; }
    if (!peers && !d_out && out_capacity) { set_error("m2s_convert: output buffer is NULL"); return M2S_E_INVALID; }
    if (peers) {
        if (peers->world < 1 || peers->world > M2S_MAX_PEERS || peers->rank >= peers->world) { set_error("m2s_convert_gather: bad world/rank"); return M2S_E_INVALID; }
        if (p->layout > M2S_LAYOUT_PACKED56) { set_error("m2s_convert_gather: layouts REF96 and PACKED56 only"); return M2S_E_INVALID; }
        for (uint32_t r = 0; r < peers->world; ++r)
            if (!peers->out[r] || !peers->xch[r] || (reinterpret_cast<uintptr_t>(peers->out[r]) & 15u)) { set_error("m2s_convert_gather: NULL or misaligned peer buffer"); return M2S_E_INVALID; }
    }
    if (!(p->gaussian_std > 0.0f) && p->layout != M2S_LAYOUT_REF96) { set_error("m2s_convert: gaussian_std must be > 0"); return M2S_E_INVALID; }
    const TriRange tr = tri_range(p->first_triangle, p->triangle_count, s->ntri);
    CUDA_TRY(cudaSetDevice(ctx->device));
    cudaStream_t stream = pick_stream(ctx, stream_);
    const int klayout = (int)p->layout;  // every layout, the .ply rows included, is written by the fragment kernel itself
    if (!aligned_ok("m2s_convert", "the output buffer must be 16-byte aligned", {{d_out, 16}})) return M2S_E_INVALID;
    ConvertPlan pl;
    convert_plan(ctx, s, p, out_capacity, (peers && peers->world > 1) ? peers->world : 1u, &pl);
    // scratch between the two kernels (grown on demand, kept by the context)
    m2s_status st = grow(ctx, ctx->trifrag, std::max<uint64_t>(tr.count, 1) * tri_frag_bytes(klayout), stream);
    if (st == M2S_OK) st = grow(ctx, ctx->items, pl.queue_cap * sizeof(FragItem), stream);
    if (st != M2S_OK) return st;
    if (ctx->dirty) {
        CUDA_TRY(cudaMemsetAsync(ctx->d_sched, 0, 8 * 128, stream));
        CUDA_TRY(cudaMemsetAsync(ctx->d_counter, 0, sizeof(unsigned long long), stream));
        ctx->dirty = false;
    }
    ConvertArgs a;
    std::memset(&a, 0, sizeof(a));
    a.tris = s->d_tris;
    a.tri_first = (uint32_t)tr.first;
    a.tri_count = (uint32_t)tr.count;
    a.ranges = s->d_ranges; a.nranges = s->nranges;
    a.prims = s->d_prims; a.nprims = s->nprims; a.texs = s->d_texs; a.tex_base = s->d_arena; a.ntex = s->ntex;
    a.R = p->resolution;
    a.row_begin = std::min(p->row_begin, p->resolution);
    a.row_end = (p->row_end == 0 || p->row_end > p->resolution) ? p->resolution : p->row_end;
    a.half_R = (float)p->resolution * 0.5f;
    a.mult = p->gaussian_std / (float)p->resolution;
    a.log_sz = logf(1e-7f * a.mult);
    a.tri_frag = (unsigned char*)ctx->trifrag.p;
    a.items = (FragItem*)ctx->items.p;
    a.queue_cap = (uint32_t)pl.queue_cap;
    a.item_max_frags = (uint32_t)pl.item_max;
    a.flush_frags = (uint32_t)pl.flush_frags;
    a.n_items_out = ctx->d_nitems;
    a.out = (uint8_t*)d_out;
    a.cap = pl.cap;
    a.keys = (unsigned long long*)d_keys;
    a.counter = ctx->d_counter;
    // fused gather: the raster kernel's count stays local, the global total goes to d_total after the wait
    a.total_out = (peers && peers->world > 1) ? ctx->d_total : (d_total ? (unsigned long long*)d_total : ctx->d_total);
    a.prev_totals = prev_totals;
    a.nprev = nprev;
    a.host_total = host_total;
    a.host_tag = host_tag;
    a.sched = ctx->d_sched;
    a.unit_tris = (uint32_t)pl.unit_tris;
    a.n_units = (uint32_t)pl.n_units;
    a.direct_ok = (uint32_t)pl.direct_ok;
    a.claim_late = (uint32_t)pl.claim_late;
    a.trace = g_trace;
    if (peers && peers->world > 1) {
        a.world = peers->world; a.rank = peers->rank;
        for (uint32_t r = 0; r < peers->world; ++r) { a.peer_out[r] = (uint8_t*)peers->out[r]; a.peer_xch[r] = (unsigned long long*)peers->xch[r]; }
        a.epoch = ++ctx->epoch;
        a.gcap = out_capacity;
        a.status = ctx->d_status;
    }
    const int fgrid = ctx->sm_count * ctx->frag_blocks_per_sm[klayout];
    cudaError_t e = convert_launch(klayout, a, (int)pl.grid, fgrid, stream, mid);
    if (e != cudaSuccess) { ctx->dirty = true; set_error(std::string("convert launch: ") + cudaGetErrorString(e)); return M2S_E_CUDA; }
    if (peers && peers->world > 1)
        CUDA_TRY(gather_wait_launch((const unsigned long long*)peers->xch[peers->rank], peers->world, a.epoch, out_capacity,
                                    (unsigned long long*)d_total, ctx->d_status, stream));
    return M2S_OK;
}

M2S_EXPORT m2s_status m2s_convert_enqueue(m2s_ctx* ctx, const m2s_dscene* s, const m2s_params* p, void* d_out,
                                          uint64_t out_capacity, uint64_t* d_keys, uint64_t* d_total, void* stream_) {
    return convert_enqueue_impl(ctx, s, p, d_out, out_capacity, d_keys, d_total, stream_, nullptr);
}

M2S_EXPORT m2s_status m2s_convert_gather_enqueue(m2s_ctx* ctx, const m2s_dscene* s, const m2s_params* p, const m2s_peers* peers,
                                                 uint64_t out_capacity, uint64_t* d_total_global, void* stream_) {
    if (!peers) { set_error("m2s_convert_gather: peers is NULL"); return M2S_E_INVALID; }
    if (peers->world <= 1)  // degenerate: plain conversion into the local final buffer
        return convert_enqueue_impl(ctx, s, p, peers->out[0], out_capacity, nullptr, d_total_global, stream_, nullptr);
    return convert_enqueue_impl(ctx, s, p, nullptr, out_capacity, nullptr, d_total_global, stream_, peers);
}

M2S_EXPORT m2s_status m2s_convert(m2s_ctx* ctx, const m2s_dscene* s, const m2s_params* p, void* d_out, uint64_t out_capacity,
                                  uint64_t* d_keys, m2s_result* res) {
    if (!ctx) { set_error("m2s_convert: ctx is NULL"); return M2S_E_INVALID; }
    CUDA_TRY(cudaSetDevice(ctx->device));
    CUDA_TRY(cudaEventRecord(ctx->ev0, ctx->stream));
    m2s_status st = m2s_convert_enqueue(ctx, s, p, d_out, out_capacity, d_keys, nullptr, ctx->stream);
    if (st != M2S_OK) return st;
    CUDA_TRY(cudaEventRecord(ctx->ev1, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(ctx->h_total, ctx->d_total, sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx->stream));
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { ctx->dirty = true; set_error(std::string("convert: ") + cudaGetErrorString(e)); return M2S_E_CUDA; }
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1);
    const uint64_t cap = effective_cap(s, p, out_capacity);
    const uint64_t total = *ctx->h_total;
    if (res) { res->total = total; res->cap = cap; res->written = std::min(total, cap); res->device_ms = ms; }
    return total > cap ? capacity_error(total, cap) : M2S_OK;
}

// Measurement aid: one conversion with an event between the two kernels (no programmatic dependent launch, so they do
// not overlap): the per-kernel shares of the step, measured live instead of read from a profile.
M2S_EXPORT m2s_status m2s_convert_timed(m2s_ctx* ctx, const m2s_dscene* s, const m2s_params* p, void* d_out, uint64_t out_capacity,
                                        float* raster_ms, float* fragment_ms) {
    if (!ctx) { set_error("m2s_convert_timed: ctx is NULL"); return M2S_E_INVALID; }
    CUDA_TRY(cudaSetDevice(ctx->device));
    if (!ctx->ev_mid) CUDA_TRY(cudaEventCreate(&ctx->ev_mid));
    CUDA_TRY(cudaEventRecord(ctx->ev0, ctx->stream));
    m2s_status st = convert_enqueue_impl(ctx, s, p, d_out, out_capacity, nullptr, nullptr, ctx->stream, nullptr, nullptr, 0, nullptr, 0, ctx->ev_mid);
    if (st != M2S_OK) return st;
    CUDA_TRY(cudaEventRecord(ctx->ev1, ctx->stream));
    cudaError_t e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) { ctx->dirty = true; set_error(std::string("convert_timed: ") + cudaGetErrorString(e)); return M2S_E_CUDA; }
    float a = 0.f, b = 0.f;
    cudaEventElapsedTime(&a, ctx->ev0, ctx->ev_mid);
    cudaEventElapsedTime(&b, ctx->ev_mid, ctx->ev1);
    if (raster_ms) *raster_ms = a;
    if (fragment_ms) *fragment_ms = b;
    return M2S_OK;
}

M2S_EXPORT m2s_status m2s_convert_host(m2s_ctx* ctx, const m2s_scene* sc, const m2s_params* p, void* h_out, uint64_t out_capacity,
                                       uint64_t* h_keys, m2s_result* res) {
    if (!ctx || !sc || !p || (!h_out && out_capacity)) { set_error("m2s_convert_host: NULL argument"); return M2S_E_INVALID; }
    const uint32_t stride = m2s_record_stride(p->layout);
    if (!stride) { set_error("m2s_convert_host: unknown layout"); return M2S_E_INVALID; }
    CUDA_TRY(cudaSetDevice(ctx->device));
    SlimScene slim_holder(sc, p->layout);
    const m2s_scene& slim = slim_holder.scene;
    // Pipeline (REF96 / PACKED56, meshes large enough to split): the triangle range is cut into chunks; chunk c's
    // records are appended after chunk c-1's on the device (fragment kernel: prev_totals) and start crossing
    // PCIe on a second stream while chunk c+1 is still being uploaded and converted — H2D and D2H overlap.
    const TriRange tr = tri_range(p->first_triangle, p->triangle_count, sc->triangle_count);
    const uint64_t first = tr.first, count = tr.count;
    int nchunks = 1;
    if (count >= 16384) {  // every layout: the fragment kernel appends after the earlier chunks' records itself
        // every chunk shortens the tail (the last chunk's kernels and download) and costs ~25 us of kernel latency on the
        // compute stream, hidden behind the uploads; chunks of >= 8 k triangles keep the GPU filled
        nchunks = (int)std::max<uint64_t>(2, std::min<uint64_t>(4, count / 16384));
        if (const char* e = std::getenv("M2S_HOST_CHUNKS")) nchunks = std::max(1, std::min(m2s_ctx::kMaxChunks, std::atoi(e)));
    }
    const uint64_t per = (count + nchunks - 1) / nchunks;
    m2s_dscene* ds = nullptr;
    // Pipeline: (1) the triangle chunks go up back to back, each followed by a reduction of its v-range per texture and
    // a 8-byte-per-texture copy back; (2) per chunk, as soon as its v-range is on the host: the texture row groups it
    // samples (not yet resident) go up, the two kernels are enqueued; (3) a chunk's records start crossing PCIe on a
    // second stream as soon as its count has arrived (zero-copy, from the raster kernel's last CTA) while later chunks
    // are still being uploaded and converted.  The first records exist after ~1/nchunks of the upload; a shard
    // (first_triangle/triangle_count) never uploads texture rows it does not sample.
    m2s_status st = scene_upload_impl(ctx, &slim, &ds, 0, false, first, true);
    if (st != M2S_OK) return st;
    st = grow(ctx, ctx->out, std::max<uint64_t>(out_capacity, 1) * stride);
    if (st == M2S_OK && h_keys) st = grow(ctx, ctx->keys, std::max<uint64_t>(out_capacity, 1) * 8);
    if (st != M2S_OK) { cudaStreamSynchronize(ctx->stream); m2s_scene_free(ctx, ds); return st; }
    unsigned long long* const d_keys = static_cast<unsigned long long*>(ctx->keys.p);
    m2s_result r;
    std::memset(&r, 0, sizeof(r));
    const uint64_t cap = effective_cap(ds, p, out_capacity);
    auto fail_with = [&](m2s_status code) {
        cudaStreamSynchronize(ctx->stream3); cudaStreamSynchronize(ctx->stream4); cudaStreamSynchronize(ctx->stream5);
        cudaStreamSynchronize(ctx->stream); cudaStreamSynchronize(ctx->stream2);
        ctx->dirty = true; ctx->vr_dirty = true;
        m2s_scene_free(ctx, ds);
        return code;
    };
    auto bail = [&](const char* what, cudaError_t e) {
        set_error(std::string(what) + ": " + cudaGetErrorString(e));
        return fail_with(M2S_E_CUDA);
    };
    static const bool host_trace = std::getenv("M2S_HOST_TRACE") != nullptr;  // debug: phase times on stderr
    const auto t_start = std::chrono::steady_clock::now();
    auto since = [&]() { return std::chrono::duration<double, std::micro>(std::chrono::steady_clock::now() - t_start).count(); };
    cudaError_t e = cudaEventRecord(ctx->ev0, ctx->stream);
    if (e != cudaSuccess) return bail("convert_host", e);
    // uploads run on their own stream (behind the allocations and table copies made above on the context stream): the
    // copy engine streams triangles and texture rows continuously while the chunks' kernels run on the context stream
    e = cudaEventRecord(ctx->ev_alloc, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(ctx->stream3, ctx->ev_alloc, 0);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(ctx->stream4, ctx->ev_alloc, 0);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(ctx->stream5, ctx->ev_alloc, 0);
    if (e != cudaSuccess) return bail("convert_host", e);
    // triangles on one copy stream, texture rows on another (two copy engines), the v-range
    // reductions on a third, the mip rows on the compute stream: no copy ever queues behind a kernel
    struct UpGuard { m2s_ctx* c; ~UpGuard() { c->up = c->tex_up = c->mip = c->aux = c->stream; } } up_guard{ctx};
    ctx->up = ctx->stream3; ctx->tex_up = ctx->stream4; ctx->aux = ctx->stream5; ctx->mip = ctx->stream;
    uint64_t lo_[m2s_ctx::kMaxChunks], hi_[m2s_ctx::kMaxChunks];
    int planned = 0, uploaded = 0;
    for (int c = 0; c < nchunks; ++c) {
        const uint64_t lo = first + (uint64_t)c * per, hi = std::min(first + count, lo + per);
        if (lo >= hi && c > 0) break;
        lo_[c] = lo; hi_[c] = hi;
        ++planned;
    }
    // (1) triangle chunk c goes up (its own copy stream), followed by the reduction of its v-range per texture (a kernel behind
    // "chunk c is resident" on the aux stream, results through mapped memory)
    auto upload_tris = [&](int c) -> m2s_status {
        cudaError_t e1 = cudaSuccess;
        if (hi_[c] > lo_[c]) {
            e1 = cudaMemcpyAsync(reinterpret_cast<unsigned char*>(ds->d_tris) + lo_[c] * (size_t)kTriBytes,
                                 reinterpret_cast<const unsigned char*>(sc->triangles) + lo_[c] * (size_t)kTriBytes,
                                 (hi_[c] - lo_[c]) * (size_t)kTriBytes, cudaMemcpyHostToDevice, ctx->up);
            ds->h2d_bytes += (hi_[c] - lo_[c]) * (uint64_t)kTriBytes;
        }
        if (e1 == cudaSuccess) e1 = cudaEventRecord(ctx->ev_tri[c], ctx->up);
        if (e1 == cudaSuccess) e1 = cudaStreamWaitEvent(ctx->aux, ctx->ev_tri[c], 0);
        if (e1 != cudaSuccess) { set_error(std::string("convert_host upload: ") + cudaGetErrorString(e1)); return M2S_E_CUDA; }
        return vrange_enqueue(ctx, ds, lo_[c], hi_[c], c);
    };
    // look-ahead: triangle chunks (and their v-range reductions) queued ahead of the chunk whose texture rows go up: the
    // first records exist after ~lookahead/nchunks of the triangles and 1/nchunks of the texture rows (the downloads of the
    // records are the longest leg of the call: they must start early; queueing every triangle chunk up front delays them)
    int lookahead = 2;
    if (const char* e = std::getenv("M2S_HOST_LOOKAHEAD")) lookahead = std::max(1, std::atoi(e));
    for (; uploaded < std::min(planned, lookahead); ++uploaded) {
        st = upload_tris(uploaded);
        if (st != M2S_OK) return fail_with(st);
    }
    unsigned long long tags[m2s_ctx::kMaxChunks] = {};
    uint64_t base = 0, written = 0;
    int next_dl = 0;
    // enqueue the downloads of the chunks whose counts have arrived (in order); block: wait for them
    auto downloads = [&](int upto, bool block) -> cudaError_t {
        while (next_dl < upto) {
            const int c = next_dl;
            volatile unsigned long long* slot = ctx->h_chunk_tot + 2 * c;
            for (;;) {
                if (__atomic_load_n(&ctx->h_chunk_tot[2 * c + 1], __ATOMIC_ACQUIRE) == tags[c]) break;  // count is ordered before the tag
                if (!block) return cudaSuccess;
                const cudaError_t q = cudaEventQuery(ctx->ev_chunk[c]);
                if (q == cudaSuccess) break;             // finished: the tag is there
                if (q != cudaErrorNotReady) return q;
            }
            if (__atomic_load_n(&ctx->h_chunk_tot[2 * c + 1], __ATOMIC_ACQUIRE) != tags[c]) return cudaErrorUnknown;
            const uint64_t tot = slot[0];
            if (host_trace) std::fprintf(stderr, "[m2s host] chunk %d rasterised at %.0f us (%llu records)\n", c, since(), (unsigned long long)tot);
            const uint64_t room = cap > base ? cap - base : 0, w = std::min(tot, room);
            if (w) {
                cudaError_t e2 = cudaStreamWaitEvent(ctx->stream2, ctx->ev_chunk[c], 0);
                if (e2 == cudaSuccess)
                    e2 = cudaMemcpyAsync(reinterpret_cast<unsigned char*>(h_out) + base * stride,
                                         reinterpret_cast<const unsigned char*>(ctx->out.p) + base * stride, w * stride,
                                         cudaMemcpyDeviceToHost, ctx->stream2);
                if (e2 == cudaSuccess && h_keys)
                    e2 = cudaMemcpyAsync(h_keys + base, d_keys + base, w * 8, cudaMemcpyDeviceToHost, ctx->stream2);
                if (e2 != cudaSuccess) return e2;
            }
            base += tot;
            written += w;
            ++next_dl;
        }
        return cudaSuccess;
    };
    int launched = 0;
    for (int c = 0; c < planned; ++c) {  // (2)
        std::vector<MipRun> runs;
        const double t_it0 = host_trace ? since() : 0.0;
        st = upload_groups_from_vrange(ctx, ds, c, [&] { return downloads(launched, false); }, &runs);  // (3) while waiting: whatever is ready
        if (st != M2S_OK) return fail_with(st);
        const double t_it1 = host_trace ? since() : 0.0;
        e = cudaEventRecord(ctx->ev_up[c], ctx->tex_up);   // chunk c's texture rows are resident (level 0)
        if (e == cudaSuccess) e = cudaStreamWaitEvent(ctx->stream, ctx->ev_up[c], 0);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(ctx->stream, ctx->ev_tri[c], 0);
        if (e != cudaSuccess) return bail("convert_host", e);
        for (const MipRun& r : runs) {   // their mip rows: on the compute stream, right before the kernels that sample them
            e = mip_groups_launch(ds->d_arena, ds->h_texs[r.t], r.g0, r.g1, ctx->stream);
            if (e != cudaSuccess) return bail("convert_host mips", e);
        }
        if (uploaded < planned) {  // the next look-ahead chunk
            st = upload_tris(uploaded++);
            if (st != M2S_OK) return fail_with(st);
        }
        m2s_params pc = *p;
        pc.first_triangle = lo_[c];
        pc.triangle_count = hi_[c] - lo_[c];
        unsigned long long* h_dev = nullptr;  // device view of the mapped count slot
        e = cudaHostGetDevicePointer((void**)&h_dev, ctx->h_chunk_tot + 2 * c, 0);
        if (e != cudaSuccess) return bail("convert_host", e);
        tags[c] = ++ctx->host_seq;
        if (hi_[c] > lo_[c]) {
            st = convert_enqueue_impl(ctx, ds, &pc, ctx->out.p, out_capacity, h_keys ? (uint64_t*)d_keys : nullptr,
                                      (uint64_t*)(ctx->d_chunk_tot + c), ctx->stream, nullptr, ctx->d_chunk_tot, (uint32_t)c,
                                      h_dev, tags[c]);
            if (st != M2S_OK) return fail_with(st);
        } else {  // empty range: nothing to launch, the count is zero
            e = cudaMemsetAsync(ctx->d_chunk_tot + c, 0, sizeof(unsigned long long), ctx->stream);
            if (e != cudaSuccess) return bail("convert_host", e);
            ctx->h_chunk_tot[2 * c] = 0;
            __atomic_store_n(&ctx->h_chunk_tot[2 * c + 1], tags[c], __ATOMIC_RELEASE);
        }
        e = cudaEventRecord(ctx->ev_chunk[c], ctx->stream);
        if (e != cudaSuccess) return bail("convert_host", e);
        ++launched;
        const double t_it2 = host_trace ? since() : 0.0;
        e = downloads(launched, false);  // (3) whatever is ready
        if (e != cudaSuccess) return bail("convert_host download", e);
        if (host_trace) std::fprintf(stderr, "[m2s host] chunk %d: v-range wait + rows enqueued %.0f us, tris/mips/kernels enqueued %.0f us, downloads %.0f us (at %.0f us)\n",
                                     c, t_it1 - t_it0, t_it2 - t_it1, since() - t_it2, since());
    }
    e = cudaEventRecord(ctx->ev1, ctx->stream);
    if (e != cudaSuccess) return bail("convert_host", e);
    if (host_trace) std::fprintf(stderr, "[m2s host] enqueued %d chunks at %.0f us\n", launched, since());
    e = downloads(launched, true);
    if (e != cudaSuccess) return bail("convert_host download", e);
    e = cudaStreamSynchronize(ctx->stream2);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream3);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream4);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream5);
    if (e != cudaSuccess) return bail("convert_host download", e);
    if (host_trace) std::fprintf(stderr, "[m2s host] downloads done at %.0f us\n", since());
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1);
    r.total = base; r.cap = cap; r.written = written; r.device_ms = ms;
    st = base > cap ? capacity_error(base, cap) : M2S_OK;
    if (res) *res = r;
    m2s_scene_free(ctx, ds);
    return st;
}

// ---- scene -> .ply file: rows encoded on the GPU, streamed to disk through two pinned buffers -------------
// (SceneManager::exportPly + parsers.cpp::savePlyVector write 4 bytes at a time from one thread)
m2s_status m2s::convert_scene_to_ply(m2s_ctx* ctx, const m2s_scene* sc, const m2s_params* p, const char* path, m2s_result* res) {
    if (!ctx || !sc || !p || !path) { set_error("convert_scene_to_ply: NULL argument"); return M2S_E_INVALID; }
    if (p->layout < M2S_LAYOUT_PLY_STANDARD || p->layout > M2S_LAYOUT_PLY_COMPRESSED) { set_error("convert_scene_to_ply: a .ply row layout is required"); return M2S_E_INVALID; }
    const uint32_t format = p->layout - M2S_LAYOUT_PLY_STANDARD;
    const uint32_t stride = m2s_record_stride(p->layout);
    CUDA_TRY(cudaSetDevice(ctx->device));
    SlimScene slim(sc, p->layout);
    m2s_dscene* ds = nullptr;
    m2s_status st = scene_upload_impl(ctx, &slim.scene, &ds, UINT64_MAX, false);
    if (st != M2S_OK) return st;
    const uint64_t cap = p->max_gaussians ? p->max_gaussians : m2s_reference_capacity(p->resolution, sc->primitive_count);
    st = grow(ctx, ctx->out, std::max<uint64_t>(cap, 1) * stride);
    if (st != M2S_OK) { cudaStreamSynchronize(ctx->stream); m2s_scene_free(ctx, ds); return st; }
    m2s_result r;
    std::memset(&r, 0, sizeof(r));
    st = m2s_convert(ctx, ds, p, ctx->out.p, cap, nullptr, &r);  // synchronises; r.written rows are in ctx->out
    m2s_scene_free(ctx, ds);
    if (res) *res = r;
    if (st != M2S_OK && st != M2S_E_CAPACITY) return st;
    for (int i = 0; i < 2; ++i)
        if (!ctx->h_stage[i]) CUDA_TRY(cudaMallocHost(&ctx->h_stage[i], m2s_ctx::kStageBytes));
    FILE* f = std::fopen(path, "wb");
    if (!f) { set_error(std::string("cannot open ") + path); return M2S_E_IO; }
    char hdr[4096];
    const size_t hn = m2s_ply_header(format, r.written, hdr, sizeof(hdr));
    bool ok = std::fwrite(hdr, 1, hn, f) == hn;
    const size_t rows_per_block = m2s_ctx::kStageBytes / stride;
    const uint64_t nblocks = (r.written + rows_per_block - 1) / rows_per_block;
    cudaError_t e = cudaSuccess;
    auto block_bytes = [&](uint64_t b) { return (size_t)std::min<uint64_t>(rows_per_block, r.written - b * rows_per_block) * stride; };
    for (uint64_t b = 0; b <= nblocks && ok && e == cudaSuccess; ++b) {
        if (b < nblocks) {  // start the download of block b ...
            e = cudaMemcpyAsync(ctx->h_stage[b & 1], reinterpret_cast<const unsigned char*>(ctx->out.p) + b * rows_per_block * stride,
                                block_bytes(b), cudaMemcpyDeviceToHost, ctx->stream);
            if (e == cudaSuccess) e = cudaEventRecord(ctx->ev_chunk[b & 1], ctx->stream);
        }
        if (b > 0 && e == cudaSuccess) {  // ... and write block b-1 while it crosses PCIe
            e = cudaEventSynchronize(ctx->ev_chunk[(b - 1) & 1]);
            if (e == cudaSuccess) ok = std::fwrite(ctx->h_stage[(b - 1) & 1], 1, block_bytes(b - 1), f) == block_bytes(b - 1);
        }
    }
    cudaStreamSynchronize(ctx->stream);
    ok = (std::fclose(f) == 0) && ok;
    if (e != cudaSuccess) { set_error(std::string("convert_scene_to_ply download: ") + cudaGetErrorString(e)); return M2S_E_CUDA; }
    if (!ok) { set_error(std::string("short write to ") + path); return M2S_E_IO; }
    return st;
}

// ---- outputs ----------------------------------------------------------------------------------
M2S_EXPORT m2s_status m2s_ply_encode(m2s_ctx* ctx, const void* d_ref96, uint64_t count, uint32_t format, float mult, void* d_rows,
                                     void* stream_) {
    if (!ctx || (count && (!d_ref96 || !d_rows))) { set_error("m2s_ply_encode: NULL argument"); return M2S_E_INVALID; }
    if (format > 2) format = 0;  // savePlyVector default branch (parsers.cpp:646-648)
    CUDA_TRY(cudaSetDevice(ctx->device));
    CUDA_TRY(ply_rows_launch(d_ref96, count, nullptr, format, mult, d_rows, pick_stream(ctx, stream_)));
    return M2S_OK;
}
