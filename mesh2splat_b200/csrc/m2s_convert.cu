// m2s_convert.cu — C-ABI implementation (include/m2s.h): the conversion.  Its launch plan, the enqueue and synchronous
// forms, the pipelined host-to-host conversion (m2s_convert_host), and the .ply outputs.
#include <cmath>
#include <cstdio>

#include "m2s_ctx.cuh"

using namespace m2s;

static unsigned long long* g_trace = nullptr;  // debugging aid for M2S_TRACE builds (scripts/trace_raster.py)
M2S_EXPORT void m2s_debug_set_trace(void* p) { g_trace = (unsigned long long*)p; }
// Test aid: conversions leave every small triangle to the fragment kernel (no direct path), the route the direct path's
// records are compared against
static bool g_direct_off = false;
M2S_EXPORT void m2s_debug_set_direct_off(int off) { g_direct_off = off != 0; }
// Test aid: PACKED56 conversions stage the 144-byte triangles even when the scene has the 64-byte position/uv stream, the
// route the slim stream's records are compared against
static bool g_slim_off = false;
M2S_EXPORT void m2s_debug_set_slim_off(int off) { g_slim_off = off != 0; }
// Test aid: conversions that could end in the raster kernel launch the fragment kernel as well, the route the single
// launch's count and records are compared against
static bool g_single_off = false;
M2S_EXPORT void m2s_debug_set_single_off(int off) { g_single_off = off != 0; }

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
    uint64_t pair_first;              // 16-triangle units; a warp's first pass sets up units 2g and 2g + 1, one per half warp
    uint64_t single_launch;           // the raster kernel alone: no work item can be queued, the count is its own (DESIGN §4)
};

// world: GPUs of a fused gather; two_kernels: the caller needs the fragment kernel's work at the end of the step (an
// appended range, the host's mapped count, the per-kernel timing)
static void convert_plan(const m2s_ctx* ctx, const m2s_dscene* s, const m2s_params* p, uint64_t out_capacity, uint32_t world,
                         bool two_kernels, ConvertPlan* pl) {
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
    pl->multi_round = pl->n_units > warps;
    pl->direct_ok = klayout == M2S_LAYOUT_PACKED56 && pl->multi_round && world <= 1 && !g_direct_off;
    // the late claim evens out the weights of the direct units when each warp gets only two of them; with more units
    // per warp they average out anyway and the claim's exposed atomic round trip is not worth it (DESIGN §4)
    pl->claim_late = pl->direct_ok && pl->n_units < 3 * warps;
    pl->direct_max = M2S_DIRECT_MAX;
    // a balanced unit of 17-24 triangles leaves 8-15 lanes of every set-up and walk idle.  With units of 16 a warp's first
    // pass sets up two of them on its 32 lanes; the units beyond the static pairs are claimed late, one at a time.  Only
    // up to 3 units of 16 per warp: a warp then runs the pair and at most one more unit on average, never more passes
    // than with the balanced units (DESIGN §4)
    pl->pair_first = pl->claim_late && count <= 3 * warps * (kUnitTris / 2);
    if (pl->pair_first) {
        pl->unit_tris = kUnitTris / 2;
        pl->n_units = (count + pl->unit_tris - 1) / pl->unit_tris;
    }
    // a launch on the direct path needs no fragment kernel when nothing can reach the queue: every triangle's candidate
    // box is small at this density (the scene's bound), and units beyond M2S_DIRECT_MAX are shaded in rounds.  The last
    // raster CTA then publishes the count
    pl->single_launch = pl->direct_ok && !two_kernels && !g_single_off && (float)p->resolution <= s->r_small_max;
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
}

// Test and tuning aid (not part of m2s.h): the plan m2s_convert would launch with for these arguments.  `plan` receives
// the fields of ConvertPlan in order.
M2S_EXPORT m2s_status m2s_debug_convert_plan(m2s_ctx* ctx, const m2s_dscene* s, const m2s_params* p, uint64_t out_capacity, uint64_t* plan) {
    if (!ctx || !s || !p || !plan) { set_error("m2s_debug_convert_plan: NULL argument"); return M2S_E_INVALID; }
    if (p->resolution < 1 || p->resolution > 4096 || p->layout > M2S_LAYOUT_PLY_COMPRESSED) { set_error("m2s_debug_convert_plan: bad params"); return M2S_E_INVALID; }
    ConvertPlan pl;
    convert_plan(ctx, s, p, out_capacity, 1u, false, &pl);
    std::memcpy(plan, &pl, sizeof(pl));
    return M2S_OK;
}

// The kernels of one conversion on one stream: the raster kernel, then the fragment kernel unless the launch is single.
// mid != nullptr: recorded between them (measurement of the per-kernel shares); the fragment kernel then launches without
// programmatic dependent launch, so the kernels do not overlap.
static cudaError_t convert_launch(int layout, const ConvertArgs& a, int raster_grid, int fragment_grid, cudaStream_t stream, cudaEvent_t mid) {
    cudaError_t e = raster_launch(layout, a, raster_grid, stream);
    if (e != cudaSuccess || a.single_launch) return e;
    if (mid) { e = cudaEventRecord(mid, stream); if (e != cudaSuccess) return e; }
    return fragment_launch(layout, a, fragment_grid, mid == nullptr, stream);
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
    convert_plan(ctx, s, p, out_capacity, (peers && peers->world > 1) ? peers->world : 1u, nprev != 0 || host_total || mid, &pl);
    // scratch between the two kernels (grown on demand, kept by the context)
    m2s_status st = grow(ctx, ctx->trifrag, std::max<uint64_t>(tr.count, 1) * tri_frag_bytes(klayout), stream);
    if (st == M2S_OK) st = grow(ctx, ctx->items, pl.queue_cap * sizeof(FragItem), stream);
    if (st != M2S_OK) return st;
    if (ctx->dirty) {  // both scheduler sets
        CUDA_TRY(cudaMemsetAsync(ctx->d_sched, 0, 8 * 128, stream));
        ctx->dirty = false;
    }
    ConvertArgs a;
    std::memset(&a, 0, sizeof(a));
    a.tris = s->d_tris;
    a.tris_slim = (klayout == M2S_LAYOUT_PACKED56 && !g_slim_off) ? s->d_tris_slim : nullptr;   // only PACKED56's set-up reads it
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
    a.out = (uint8_t*)d_out;
    a.cap = pl.cap;
    a.keys = (unsigned long long*)d_keys;
    // the scheduler set of this launch, {unit counter, packed counter} at lines {2 s, 2 s + 1} of d_sched, and the next's
    auto set_claim = [&](uint32_t s) { return ctx->d_sched + 2 * s * kSchedStride; };
    auto set_counter = [&](uint32_t s) { return reinterpret_cast<unsigned long long*>(ctx->d_sched + (2 * s + 1) * kSchedStride); };
    a.claim = set_claim(ctx->sched_parity);
    a.counter = set_counter(ctx->sched_parity);
    a.next_claim = set_claim(ctx->sched_parity ^ 1u);
    a.next_counter = set_counter(ctx->sched_parity ^ 1u);
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
    a.pair_first = (uint32_t)pl.pair_first;
    a.single_launch = (uint32_t)pl.single_launch;
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
    ctx->sched_parity ^= 1u;   // this launch's raster kernel zeroes the other set
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
// not overlap): the per-kernel shares of the step, measured live instead of read from a profile.  Always both kernels,
// also where m2s_convert would end in the raster kernel, so the two shares keep their meaning.
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

// ---- host buffers in, host buffers out: the pipelined conversion ------------------------------------------------------
m2s_status m2s::HostPipeline::create() {
    for (cudaStream_t* s : {&tri_stream, &tex_stream, &vr_stream, &dl_stream}) CUDA_TRY(cudaStreamCreateWithFlags(s, cudaStreamNonBlocking));
    CUDA_TRY(cudaEventCreateWithFlags(&ev_alloc, cudaEventDisableTiming));
    for (int i = 0; i < kMaxChunks; ++i)
        for (cudaEvent_t* ev : {&ev_tri[i], &ev_up[i], &ev_chunk[i]}) CUDA_TRY(cudaEventCreateWithFlags(ev, cudaEventDisableTiming));
    CUDA_TRY(cudaMalloc(&d_chunk_tot, kMaxChunks * sizeof(unsigned long long)));
    CUDA_TRY(cudaHostAlloc(&h_chunk_tot, 2 * kMaxChunks * sizeof(unsigned long long), cudaHostAllocMapped));
    std::memset(h_chunk_tot, 0, 2 * kMaxChunks * sizeof(unsigned long long));
    return M2S_OK;
}

void m2s::HostPipeline::release() {
    cudaFree(d_chunk_tot);
    if (h_chunk_tot) cudaFreeHost(h_chunk_tot);
    for (VRangeSlot& v : vr) { if (v.d_minmax) cudaFree(v.d_minmax); if (v.h_minmax) cudaFreeHost(v.h_minmax); if (v.ev) cudaEventDestroy(v.ev); }
    for (int i = 0; i < kMaxChunks; ++i)
        for (cudaEvent_t ev : {ev_tri[i], ev_up[i], ev_chunk[i]}) if (ev) cudaEventDestroy(ev);
    if (ev_alloc) cudaEventDestroy(ev_alloc);
    for (cudaStream_t s : {tri_stream, tex_stream, vr_stream, dl_stream}) if (s) cudaStreamDestroy(s);
}

namespace {

constexpr int kMaxChunks = HostPipeline::kMaxChunks;
// triangle chunks (and their v-range reductions) queued ahead of the chunk whose texture rows go up: the first records
// exist after ~kLookahead/nchunks of the triangles and 1/nchunks of the texture rows (the downloads of the records are
// the longest leg of the call: they must start early; queueing every triangle chunk up front delays them)
constexpr int kLookahead = 2;

// M2S_OK, or M2S_E_CUDA with the error "<what>: <e>"
m2s_status cuda_status(const char* what, cudaError_t e) {
    if (e == cudaSuccess) return M2S_OK;
    set_error(std::string(what) + ": " + cudaGetErrorString(e));
    return M2S_E_CUDA;
}

// One m2s_convert_host call: a pipeline over the chunks of its triangle range.  Chunk c's records are appended after
// chunk c-1's on the device (the fragment kernel adds the earlier chunks' counts, prev_totals).  (1) The triangle chunks
// go up back to back on the triangle stream, kLookahead ahead of the chunk being converted, each followed on the v-range
// stream by the reduction of its v-range per texture and an 8-byte-per-texture copy back.  (2) Per chunk, as soon as its
// v-range is on the host: the texture row groups it samples (not yet resident) go up on the texture stream, and the
// compute stream (the context's) generates their mip rows and runs the two kernels.  (3) A chunk's records start
// crossing PCIe on the download stream as soon as its count has arrived (zero-copy, from the fragment kernel as it starts),
// while later chunks are still being uploaded and converted.  The first records exist after ~1/nchunks of the upload; a
// shard (first_triangle/triangle_count) never uploads texture rows it does not sample.
struct HostConvert {
    m2s_ctx* ctx;
    HostPipeline& hp;                           // ctx->pipeline
    const m2s_scene* sc;                        // the call's arguments
    const m2s_params* p;
    unsigned char* h_out;
    uint64_t* h_keys;
    uint64_t out_capacity;
    uint32_t stride;                            // record bytes of p->layout
    m2s_dscene* ds = nullptr;
    uint64_t cap = 0;                           // the effective cap
    uint64_t first = 0, end = 0, per = 0;       // the triangle range [first, end), in chunks of `per` triangles
    int nchunks = 0, uploaded = 0, launched = 0, downloaded = 0;  // chunks planned; with triangles, kernels, downloads enqueued
    unsigned long long tags[kMaxChunks] = {};   // the tag each chunk's count arrives with
    uint64_t base = 0, written = 0;             // records of the downloaded chunks: generated, and stored

    uint64_t lo(int c) const { return first + (uint64_t)c * per; }
    uint64_t hi(int c) const { return std::min(end, lo(c) + per); }

    // the chunk plan: under 16384 triangles one chunk, otherwise count / 16384 chunks, 2 to 4.  Every chunk shortens the
    // tail (the last chunk's kernels and download) and costs ~25 us of kernel latency on the compute stream, hidden behind
    // the uploads; chunks of >= 8 k triangles keep the GPU filled.  No chunk is empty unless the range is.
    void plan(const TriRange& tr) {
        first = tr.first;
        end = tr.first + tr.count;
        nchunks = tr.count < 16384 ? 1 : (int)std::clamp<uint64_t>(tr.count / 16384, 2, kMaxChunks);
        per = (tr.count + nchunks - 1) / nchunks;
    }

    // the start event, and the upload streams behind the allocations and table copies made on the compute stream
    m2s_status start() {
        cudaError_t e = cudaEventRecord(ctx->ev0, ctx->stream);
        if (e == cudaSuccess) e = cudaEventRecord(hp.ev_alloc, ctx->stream);
        for (cudaStream_t s : {hp.tri_stream, hp.tex_stream, hp.vr_stream})
            if (e == cudaSuccess) e = cudaStreamWaitEvent(s, hp.ev_alloc, 0);
        return cuda_status("convert_host", e);
    }

    // (1) chunk c's triangles, then the reduction of its v-range behind "chunk c is resident"
    m2s_status upload_tris(int c) {
        const uint64_t n = hi(c) - lo(c);
        cudaError_t e = cudaSuccess;
        if (n) {
            e = cudaMemcpyAsync(reinterpret_cast<unsigned char*>(ds->d_tris) + lo(c) * (size_t)kTriBytes,
                                reinterpret_cast<const unsigned char*>(sc->triangles) + lo(c) * (size_t)kTriBytes,
                                n * (size_t)kTriBytes, cudaMemcpyHostToDevice, hp.tri_stream);
            ds->h2d_bytes += n * (uint64_t)kTriBytes;
        }
        if (e == cudaSuccess) e = cudaEventRecord(hp.ev_tri[c], hp.tri_stream);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(hp.vr_stream, hp.ev_tri[c], 0);
        if (e != cudaSuccess) return cuda_status("convert_host upload", e);
        return vrange_enqueue(ctx, ds, hp.vr_stream, lo(c), hi(c), c);
    }

    // (2) chunk c's texture rows once its v-range has arrived (the downloads that are ready are enqueued meanwhile), then
    // their mip rows on the compute stream, behind the rows and the chunk's triangles
    m2s_status texture_rows(int c) {
        std::vector<MipRun> runs;
        const m2s_status st = upload_groups_from_vrange(ctx, ds, hp.tex_stream, c, [&] { return downloads(false); }, &runs);
        if (st != M2S_OK) return st;
        cudaError_t e = cudaEventRecord(hp.ev_up[c], hp.tex_stream);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(ctx->stream, hp.ev_up[c], 0);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(ctx->stream, hp.ev_tri[c], 0);
        if (e != cudaSuccess) return cuda_status("convert_host", e);
        for (const MipRun& r : runs) {
            e = mip_groups_launch(ds->d_arena, ds->h_texs[r.t], r.g0, r.g1, ctx->stream);
            if (e != cudaSuccess) return cuda_status("convert_host mips", e);
        }
        return M2S_OK;
    }

    // (2) chunk c's kernels, appending after the earlier chunks' records; the count reaches its mapped slot with a fresh tag
    m2s_status launch(int c) {
        unsigned long long* h_dev = nullptr;  // device view of the mapped count slot
        cudaError_t e = cudaHostGetDevicePointer((void**)&h_dev, hp.h_chunk_tot + 2 * c, 0);
        if (e != cudaSuccess) return cuda_status("convert_host", e);
        tags[c] = ++hp.host_seq;
        if (hi(c) > lo(c)) {
            m2s_params pc = *p;
            pc.first_triangle = lo(c);
            pc.triangle_count = hi(c) - lo(c);
            const m2s_status st = convert_enqueue_impl(ctx, ds, &pc, ctx->out.p, out_capacity, h_keys ? (uint64_t*)ctx->keys.p : nullptr,
                                                       (uint64_t*)(hp.d_chunk_tot + c), ctx->stream, nullptr, hp.d_chunk_tot,
                                                       (uint32_t)c, h_dev, tags[c]);
            if (st != M2S_OK) return st;
        } else {  // empty range: nothing to launch, the count is zero
            e = cudaMemsetAsync(hp.d_chunk_tot + c, 0, sizeof(unsigned long long), ctx->stream);
            if (e != cudaSuccess) return cuda_status("convert_host", e);
            hp.h_chunk_tot[2 * c] = 0;
            __atomic_store_n(&hp.h_chunk_tot[2 * c + 1], tags[c], __ATOMIC_RELEASE);
        }
        e = cudaEventRecord(hp.ev_chunk[c], ctx->stream);
        if (e != cudaSuccess) return cuda_status("convert_host", e);
        ++launched;
        return M2S_OK;
    }

    // (3) the downloads of the launched chunks whose counts have arrived, in order; block: wait for every count
    m2s_status downloads(bool block) {
        for (; downloaded < launched; ++downloaded) {
            const int c = downloaded;
            volatile unsigned long long* slot = hp.h_chunk_tot + 2 * c;
            for (;;) {
                if (__atomic_load_n(&hp.h_chunk_tot[2 * c + 1], __ATOMIC_ACQUIRE) == tags[c]) break;  // count is ordered before the tag
                if (!block) return M2S_OK;
                const cudaError_t q = cudaEventQuery(hp.ev_chunk[c]);
                if (q == cudaSuccess) break;             // finished: the tag is there
                if (q != cudaErrorNotReady) return cuda_status("convert_host download", q);
            }
            if (__atomic_load_n(&hp.h_chunk_tot[2 * c + 1], __ATOMIC_ACQUIRE) != tags[c]) return cuda_status("convert_host download", cudaErrorUnknown);
            const uint64_t tot = slot[0];
            const uint64_t room = cap > base ? cap - base : 0, w = std::min(tot, room);
            if (w) {
                cudaError_t e = cudaStreamWaitEvent(hp.dl_stream, hp.ev_chunk[c], 0);
                if (e == cudaSuccess)
                    e = cudaMemcpyAsync(h_out + base * stride, reinterpret_cast<const unsigned char*>(ctx->out.p) + base * stride, w * stride,
                                        cudaMemcpyDeviceToHost, hp.dl_stream);
                if (e == cudaSuccess && h_keys)
                    e = cudaMemcpyAsync(h_keys + base, static_cast<const uint64_t*>(ctx->keys.p) + base, w * 8, cudaMemcpyDeviceToHost, hp.dl_stream);
                if (e != cudaSuccess) return cuda_status("convert_host download", e);
            }
            base += tot;
            written += w;
        }
        return M2S_OK;
    }

    // the stop event, every download, and every stream idle
    m2s_status drain() {
        m2s_status st = cuda_status("convert_host", cudaEventRecord(ctx->ev1, ctx->stream));
        if (st == M2S_OK) st = downloads(true);
        if (st != M2S_OK) return st;
        cudaError_t e = cudaSuccess;
        for (cudaStream_t s : {hp.dl_stream, ctx->stream, hp.tri_stream, hp.tex_stream, hp.vr_stream})
            if (e == cudaSuccess) e = cudaStreamSynchronize(s);
        return cuda_status("convert_host download", e);
    }

    // the one failure path once the streams have work: all five streams are idle before the scene is freed, and the next
    // call resets the scheduler state and re-arms the v-range slots
    m2s_status fail(m2s_status st) {
        for (cudaStream_t s : {hp.tri_stream, hp.tex_stream, hp.vr_stream, ctx->stream, hp.dl_stream}) cudaStreamSynchronize(s);
        ctx->dirty = true;
        hp.vr_dirty = true;
        m2s_scene_free(ctx, ds);
        return st;
    }
};

}  // namespace

M2S_EXPORT m2s_status m2s_convert_host(m2s_ctx* ctx, const m2s_scene* sc, const m2s_params* p, void* h_out, uint64_t out_capacity,
                                       uint64_t* h_keys, m2s_result* res) {
    if (!ctx || !sc || !p || (!h_out && out_capacity)) { set_error("m2s_convert_host: NULL argument"); return M2S_E_INVALID; }
    const uint32_t stride = m2s_record_stride(p->layout);
    if (!stride) { set_error("m2s_convert_host: unknown layout"); return M2S_E_INVALID; }
    CUDA_TRY(cudaSetDevice(ctx->device));
    HostConvert hc{ctx, ctx->pipeline, sc, p, static_cast<unsigned char*>(h_out), h_keys, out_capacity, stride};
    // the tables on the compute stream; the triangles and the texture rows come with the chunks
    const SlimScene slim(sc, p->layout);
    const TriRange tr = tri_range(p->first_triangle, p->triangle_count, sc->triangle_count);
    m2s_status st = scene_upload_impl(ctx, &slim.scene, &hc.ds, 0, false, tr.first, true);
    if (st != M2S_OK) return st;
    st = grow(ctx, ctx->out, std::max<uint64_t>(out_capacity, 1) * stride);
    if (st == M2S_OK && h_keys) st = grow(ctx, ctx->keys, std::max<uint64_t>(out_capacity, 1) * 8);
    if (st != M2S_OK) { cudaStreamSynchronize(ctx->stream); m2s_scene_free(ctx, hc.ds); return st; }
    hc.cap = effective_cap(hc.ds, p, out_capacity);
    hc.plan(tr);
    st = hc.start();
    while (st == M2S_OK && hc.uploaded < std::min(hc.nchunks, kLookahead)) st = hc.upload_tris(hc.uploaded++);
    for (int c = 0; st == M2S_OK && c < hc.nchunks; ++c) {
        st = hc.texture_rows(c);
        if (st == M2S_OK && hc.uploaded < hc.nchunks) st = hc.upload_tris(hc.uploaded++);  // the next look-ahead chunk
        if (st == M2S_OK) st = hc.launch(c);
        if (st == M2S_OK) st = hc.downloads(false);  // whatever is ready
    }
    if (st == M2S_OK) st = hc.drain();
    if (st != M2S_OK) return hc.fail(st);
    m2s_result r;
    std::memset(&r, 0, sizeof(r));
    cudaEventElapsedTime(&r.device_ms, ctx->ev0, ctx->ev1);
    r.total = hc.base; r.cap = hc.cap; r.written = hc.written;
    if (res) *res = r;
    m2s_scene_free(ctx, hc.ds);
    return hc.base > hc.cap ? capacity_error(hc.base, hc.cap) : M2S_OK;
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
            if (e == cudaSuccess) e = cudaEventRecord(ctx->ev_stage[b & 1], ctx->stream);
        }
        if (b > 0 && e == cudaSuccess) {  // ... and write block b-1 while it crosses PCIe
            e = cudaEventSynchronize(ctx->ev_stage[(b - 1) & 1]);
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
    const char* fn = "m2s_ply_encode";
    if (!ctx || (count && (!d_ref96 || !d_rows))) return invalid(fn, "NULL argument");
    if (!aligned_ok(fn, "the record and row buffers must be 16-byte aligned", {{d_ref96, 16}, {d_rows, 16}})) return M2S_E_INVALID;
    if (format > 2) format = 0;  // savePlyVector default branch (parsers.cpp:646-648)
    CUDA_TRY(cudaSetDevice(ctx->device));
    CUDA_TRY(ply_rows_launch(d_ref96, count, format, mult, d_rows, pick_stream(ctx, stream_)));
    return M2S_OK;
}
