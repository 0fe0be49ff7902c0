// m2s_fragment.cu — the conversion's second kernel: per-FRAGMENT work (converterFS.glsl:44-104), launched behind the
// raster kernel (m2s_raster.cu) with programmatic dependent launch; and the fused gather's final wait.
//
// fragment_kernel — a CTA of 4 warps takes one work item:
//   TMA stages the unit's records (three-map layouts: and its 144 B/triangle vertices) into shared memory, every
//   warp rebuilds the row spans of its share of the item's blocks (mask rows / m2s_span.cuh) into a prefix
//   table; then a warp takes 32 consecutive fragments = 32 consecutive output records: a search between the group's
//   first and last row gives (triangle, x, y); varyings from the planes (PACKED56) or from the staged vertices with
//   exact barycentrics (REF96, .ply rows); all texel loads of all bound maps issued back to back,
//   trilinear filter on the FMA pipe (u8->f32 by PRMT+FADD), TBN normal, encode (REF96 / PACKED56 / the three
//   .ply row formats directly); the 32 records are transposed through shared memory and written as one
//   contiguous span (16-byte body whatever the alignment of the span) — locally, or into every rank's final buffer
//   over NVLink (fused multi-GPU gather), or after the earlier chunks' records (appended launches of the host path).
#include <type_traits>
#include "m2s_ptx.cuh"
#include "m2s_shade.cuh"

#ifndef M2S_FRAG_WARPS
#define M2S_FRAG_WARPS 4
#endif
#ifndef M2S_FRAG_THREADS_P56
#define M2S_FRAG_THREADS_P56 1024   // resident fragment-kernel threads per SM for PACKED56 (register cap = 65536 / this)
#endif

namespace m2s {

constexpr int kFragWarps = M2S_FRAG_WARPS;
constexpr int kFragThreads = kFragWarps * 32;
constexpr uint32_t kSpanRows = kItemBlocks * 32;   // rows of an item's span table
constexpr uint32_t kMaxGroups = 128;               // 32-fragment groups of one item (< (item_max + flush) / 32)

// span table entry: one pixel row of one triangle of the item
//   x = fragments of the item before this row; y = first column (12 bits) | row relative to the box (12) << 12 | slot (5) << 24
template <int LAYOUT>
struct FragSmem {
    using Rec = TriRec<RCfg<Cfg<LAYOUT>::kRK>::kMaps>;
    static constexpr bool kVerts = LAYOUT != 1;                                   // PACKED56: the varyings are planes in the record
    static constexpr size_t kBufBytes = kUnitTris * (sizeof(Rec) + (kVerts ? kTriBytes : 0));   // one staged unit: records, then vertices
    static constexpr size_t kRecOff = 0;
    static constexpr size_t kTriOff = kUnitTris * sizeof(Rec);
    static constexpr size_t kSpanOff = kBufBytes;
    static constexpr size_t kGroupOff = kSpanOff + kSpanRows * 8;
    static constexpr size_t kStageAligned = (kGroupOff + (kMaxGroups + 1) * 2 + 15) & ~(size_t)15;
    static constexpr size_t kWarpStage = 32 * Cfg<LAYOUT>::kStride + 16;              // + the shift of a span that starts at an odd record
    static constexpr size_t kBytes = kStageAligned + (size_t)kFragWarps * kWarpStage;
};

// FragItem::first from the low and high words of the item's first 16 bytes, loaded as one uint4 h0: item_first(h0.x, h0.y)
__device__ __forceinline__ unsigned long long item_first(uint32_t lo, uint32_t hi) { return (unsigned long long)lo | ((unsigned long long)hi << 32); }

// A micro item (kItMicro): <= 32 fragments listed in the item itself, shaded by one warp with direct loads.  Out of line:
// the second copy of the shading code must not add to the register pressure of the main loop.
template <int LAYOUT>
__device__ __noinline__ void micro_item(const ConvertArgs& a, uint32_t it, uint4 h0, uint32_t nfr, unsigned long long base, unsigned long long room,
                                        unsigned long long goff, const uint32_t* __restrict__ texb, unsigned char* stage, int lane) {
    using Rec = typename FragSmem<LAYOUT>::Rec;
    constexpr int kStride = Cfg<LAYOUT>::kStride;
    const unsigned long long first = item_first(h0.x, h0.y);
    const uint32_t t0 = h0.z * a.unit_tris;
    const uint32_t w32 = __ldg(reinterpret_cast<const uint32_t*>((a.items + it)->blocks) + min((uint32_t)lane, nfr - 1u));  // idle lanes shadow the last fragment
    const uint32_t slot = w32 & 31u;
    const Rec* tfp = reinterpret_cast<const Rec*>(a.tri_frag) + (size_t)t0 + slot;
    const unsigned long long mrec = a.world <= 1 ? base + first : goff + first;   // first record of the span in its destination
    shade<LAYOUT>(a, *tfp, a.tris + ((size_t)a.tri_first + t0 + slot) * 9, (int)((w32 >> 5) & 63u), (int)((w32 >> 11) & 63u), texb,
                  stage + stage_shift<kStride>(mrec) + lane * kStride);
    __syncwarp();
    emit_records<kStride>(a, stage, nfr, first, base, room, a.world > 1, goff, it,
                          [&] { return fragment_key(a.tri_first + t0 + slot, tfp->meta, (w32 >> 5) & 63u, (w32 >> 11) & 63u); }, lane);
    __syncwarp();
}

// Thread 0 of CTA 0, once the raster grid has ended: the launch's count -> total_out, the host's mapped slot and (fused
// gather) every peer, before any CTA waits for the peers' counts.  Out of line: the kernel's other threads never run it.
__device__ __noinline__ void publish_counts(const ConvertArgs& a, unsigned long long tot) {
    *a.total_out = tot;
    if (a.host_total) {  // zero-copy count for the host (PCIe posted write, ~1 us): the count is ordered before its tag
        *reinterpret_cast<volatile unsigned long long*>(a.host_total) = tot;
        __threadfence_system();
        *reinterpret_cast<volatile unsigned long long*>(a.host_total + 1) = a.host_tag;
    }
    if (a.world > 1) {  // fused gather: tell every peer how many records this rank will write
        const unsigned long long mine = tot < a.cap ? tot : a.cap;
        for (uint32_t p = 0; p < a.world; ++p) a.peer_xch[p][a.rank * 4 + 0] = mine;
        __threadfence_system();
        for (uint32_t p = 0; p < a.world; ++p) st_release_sys(a.peer_xch[p] + a.rank * 4 + 1, a.epoch);
    }
}

template <int LAYOUT>
__global__ void __launch_bounds__(kFragThreads, (LAYOUT == 1 ? M2S_FRAG_THREADS_P56 : 512) / kFragThreads) fragment_kernel(const __grid_constant__ ConvertArgs a) {
    using S = FragSmem<LAYOUT>;
    using Rec = typename S::Rec;
    constexpr int kStride = Cfg<LAYOUT>::kStride;
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t bar[1];
    __shared__ unsigned long long s_goff;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint2* span = reinterpret_cast<uint2*>(smem + S::kSpanOff);
    unsigned short* gstart = reinterpret_cast<unsigned short*>(smem + S::kGroupOff);  // span row holding fragment 32 g of the item
    unsigned char* stage = smem + S::kStageAligned + (size_t)warp * S::kWarpStage;  // this warp's 32 records
    if (threadIdx.x == 0) {
        mbar_init(&bar[0], 1);
        fence_barrier_init();
    }
    __syncthreads();
    // ---- the item pipeline: header + block list of item i+1 are loaded while item i is processed ----
    struct Hdr { uint4 h0; uint2 h1; uint2 blk; };
    auto load_hdr = [&](uint32_t it, uint32_t bound) {
        Hdr h;
        h.h0 = make_uint4(0, 0, 0, 0); h.h1 = make_uint2(0, 0); h.blk = make_uint2(0xffffffffu, 0);
        if (it < bound) {
            const FragItem* q = a.items + it;
            h.h0 = __ldg(reinterpret_cast<const uint4*>(q));
            h.h1 = __ldg(reinterpret_cast<const uint2*>(q) + 2);
            if (!(h.h0.w & 0x80000000u) && (uint32_t)lane < (h.h0.w & 0xffu)) h.blk = __ldg(reinterpret_cast<const uint2*>(q->blocks + lane));
        }
        return h;
    };
    // launched with programmatic stream serialisation behind the raster kernel; on its direct path the raster warps trigger
    // this launch once they are out of units (pdl_launch_dependents), and the CTAs of this grid take the SMs as the raster
    // CTAs exit.  They wait here until the whole raster grid has completed; everything it wrote is visible after this wait
#ifdef M2S_TRACE
    if (a.trace && threadIdx.x == 0) atomicMin(a.trace + kTrFragStartNs, gtimer_ns());
#endif
    asm volatile("griddepcontrol.wait;" ::: "memory");
#ifdef M2S_TRACE
    if (a.trace && threadIdx.x == 0) atomicMin(a.trace + kTrFragWaitNs, gtimer_ns());
#endif
    // the first header is loaded together with the packed counter (one global round trip instead of two before the first
    // TMA): whatever an unused queue slot holds is discarded by the loop condition.  One read of the counter per CTA,
    // shared through shared memory: every warp of the grid reading the same word at once queues ~4 200 requests on one L2
    // line, and on the direct path this wait is the end of the step (DESIGN.md section 4)
    __shared__ unsigned long long s_packed;
    if (threadIdx.x == 0) s_packed = *reinterpret_cast<const volatile unsigned long long*>(a.counter);
    Hdr cur = load_hdr(blockIdx.x, a.queue_cap);
    __syncthreads();
    const unsigned long long packed = s_packed;
    const uint32_t nitems = min((uint32_t)(packed >> 40), a.queue_cap);   // work items queued
    if (blockIdx.x == 0 && threadIdx.x == 0) publish_counts(a, packed & kFragMask);
    const OutRange out = out_range(a);
    const unsigned long long base = out.base, room = out.room;
    // fused gather: wait for every rank's count of this epoch, my records start after the lower ranks'
    unsigned long long goff = 0;
    if (a.world > 1) {
        if (threadIdx.x == 0) {
            const unsigned long long* x = a.peer_xch[a.rank];
            unsigned long long off = 0;
            for (uint32_t r = 0; r < a.world; ++r) {
                wait_epoch(x + r * 4 + 1, a.epoch, a.status, 1u);  // bounded: see wait_epoch
                if (r < a.rank) off += *reinterpret_cast<const volatile unsigned long long*>(x + r * 4);
            }
            s_goff = off;
        }
        __syncthreads();
        goff = s_goff;
    }
    const uint32_t* __restrict__ texb = a.tex_base;
    auto live = [&](const Hdr& h) {  // uniform over the CTA: does the item emit anything?
        const unsigned long long first = item_first(h.h0.x, h.h0.y);
        return h.h1.y > h.h1.x && first + h.h1.x < room;
    };
    auto issue = [&](const Hdr& h, uint32_t buf) {  // thread 0: stage the unit's records: one TMA bulk copy
        const uint32_t t0 = h.h0.z * a.unit_tris;
        const uint32_t ntri = min(a.unit_tris, a.tri_count - t0);
        const uint32_t rb = ntri * (uint32_t)sizeof(Rec), tb = S::kVerts ? ntri * (uint32_t)kTriBytes : 0u;
        unsigned char* dst = smem + (size_t)buf * S::kBufBytes;
        fence_proxy_async();
        mbar_arrive_expect_tx(&bar[buf], rb + tb);
        tma_load_1d(dst + S::kRecOff, a.tri_frag + (size_t)t0 * sizeof(Rec), rb, &bar[buf]);
        if (S::kVerts) tma_load_1d(dst + S::kTriOff, reinterpret_cast<const unsigned char*>(a.tris) + ((size_t)a.tri_first + t0) * kTriBytes, tb, &bar[buf]);
    };
    uint32_t phase = 0;   // parity of the next completion of the staging barrier
    constexpr uint32_t buf = 0;
    // one header in flight per CTA: the other resident CTAs of the SM hide the load (a software pipeline over the queue
    // was measured: no gain, 16 more registers in the shading loop)
    for (uint32_t it = blockIdx.x; it < nitems; it += gridDim.x, cur = load_hdr(it, nitems)) {
        if (!live(cur)) continue;
        if (cur.h0.w & kItMicro) {
            // ---- micro item: <= 32 fragments listed in the item; ONE warp (round robin) shades it with direct loads of the
            // records it touches — no staged unit, no span table, no CTA barrier: four consecutive micro items are in
            // flight per CTA ----
            if ((uint32_t)warp == ((it / gridDim.x) & (kFragWarps - 1)))
                micro_item<LAYOUT>(a, it, cur.h0, cur.h1.y, base, room, goff, texb, stage, lane);
            continue;
        }
        // ---- the item: a unit's small triangles (implicit: one block per triangle) or queued row blocks ----
        const unsigned long long first = item_first(cur.h0.x, cur.h0.y);
        const uint32_t unit = cur.h0.z, fb = cur.h1.x, fe = cur.h1.y;
        const bool unit_item = (cur.h0.w & 0x80000000u) != 0;
        const uint32_t nblocks = cur.h0.w & 0xffu;
        const uint32_t bprefix = cur.blk.x, bref = cur.blk.y;  // lane b: block b of the item
        const uint32_t t0 = unit * a.unit_tris;
        const uint32_t ntri = min(a.unit_tris, a.tri_count - t0);
        if (threadIdx.x == 0) issue(cur, 0);
        const Rec* recs = reinterpret_cast<const Rec*>(smem + S::kRecOff);
        const float4* tris = reinterpret_cast<const float4*>(smem + S::kTriOff);
        mbar_wait(&bar[buf], phase);
        phase ^= 1u;
        // ---- the item's span table: one entry per pixel row, fragments-before-the-row ascending ----
        uint32_t nrows_flat;
        if (unit_item) {
            // the small triangles of the unit: thread (t, q) takes rows q, q+4, .. of triangle t; a row's place in the
            // table and its fragment prefix come straight from the record (TriRec::first) and the coverage mask
            const uint32_t t = threadIdx.x >> 2, q = threadIdx.x & 3u;
            if (kFragThreads < 128 && threadIdx.x == 0) __trap();  // the (t, q) mapping needs 4 threads per triangle
            if (t < ntri) {
                const Rec& r = recs[t];
                const unsigned box = r.box;
                if (box & kBoxSmall) {
                    const uint32_t w = box & 0x1fffu, h = (box >> 13) & 0x1fffu;
                    const unsigned long long hits = r.hits;
                    const uint32_t fr = r.first & 0xffffu, ro = r.first >> 16;
                    const unsigned long long rowmask = w >= 64 ? ~0ull : ((1ull << w) - 1ull);
                    for (uint32_t y = q; y < h; y += 4) {       // h * w <= 64
                        const unsigned long long below = y ? (hits & ((1ull << (y * w)) - 1ull)) : 0ull;
                        const unsigned long long bits = (hits >> (y * w)) & rowmask;
                        const uint32_t xl = bits ? (uint32_t)__ffsll((long long)bits) - 1u : 0u;
                        span[ro + y] = make_uint2(fr + (uint32_t)__popcll(below), xl | (y << 12) | (t << 24));
                    }
                }
            }
            const Rec& last = recs[ntri - 1];
            nrows_flat = (last.first >> 16) + ((last.box & kBoxSmall) ? ((last.box >> 13) & 0x1fffu) : 0u);
        } else {
            for (uint32_t b = warp; b < nblocks; b += kFragWarps) {  // one warp per block of <= 32 rows, one lane per row
                const uint32_t ref = __shfl_sync(0xffffffffu, bref, (int)b), bp = __shfl_sync(0xffffffffu, bprefix, (int)b);
                const uint32_t slot = ref & 31u, row_begin = (ref >> 5) & 0xfffu, nrows = (ref >> 17) & 63u;
                uint32_t n = 0;
                int xl = 0;
                if ((uint32_t)lane < nrows) {
                    int h;
                    n = span_row(row_state(recs[slot], h), (int)(row_begin + lane), xl);
                }
                const uint32_t incl = warp_inclusive_scan(n, lane);
                // rows past the block's last one repeat the block end: the table stays sorted, they are never selected
                span[b * 32 + lane] = make_uint2(bp + incl - n, (uint32_t)xl | ((row_begin + lane) << 12) | (slot << 24));
            }
            nrows_flat = nblocks * 32;
        }
        __syncthreads();
        // ---- where each 32-fragment group starts in the table: one binary search per group, all groups at once ----
        const uint32_t nfrag = fe - fb, ngroups = (nfrag + 31) / 32;
        for (uint32_t g = threadIdx.x; g <= ngroups; g += kFragThreads) {
            const uint32_t j = min(fb + g * 32, fe - 1);
            uint32_t lo = 0;
#pragma unroll
            for (int stp = (int)kSpanRows / 2; stp > 0; stp >>= 1) {
                const uint32_t c = lo + stp;
                if (c < nrows_flat && span[c].x <= j) lo = c;
            }
            gstart[g] = (unsigned short)lo;
        }
        __syncthreads();

        // ---- 32 consecutive fragments per warp step ----
        for (uint32_t g = warp; g < ngroups; g += kFragWarps) {
            const uint32_t j0 = fb + g * 32;
            const uint32_t nfr = min(32u, fe - j0);
            const uint32_t j = j0 + min((uint32_t)lane, nfr - 1);  // idle lanes shadow the last fragment
            // the row of fragment j: the last entry whose prefix is <= j, between the group's first and last row
            uint32_t lo = gstart[g];
            const uint32_t hi = gstart[g + 1];
            for (uint32_t stp = hi > lo ? (1u << (31 - __clz(hi - lo))) : 0u; stp; stp >>= 1) {  // uniform trip count
                const uint32_t c = lo + stp;
                if (c <= hi && span[c].x <= j) lo = c;
            }
            const uint2 sw = span[lo];
            const uint32_t slot = sw.y >> 24;
            const int dxi = (int)((sw.y & 0xfffu) + (j - sw.x)), dyi = (int)((sw.y >> 12) & 0xfffu);
            const Rec& tf = recs[slot];
            const unsigned long long idx0 = first + j0;  // index within this launch
            shade<LAYOUT>(a, tf, tris + slot * 9, dxi, dyi, texb, stage + stage_shift<kStride>(a.world <= 1 ? base + idx0 : goff + idx0) + lane * kStride);  // all 32 lanes (idle ones shadow the last fragment)
            __syncwarp();
            // ---- the warp's records are one contiguous span: straight vector copy ----
            emit_records<kStride>(a, stage, nfr, idx0, base, room, a.world > 1, goff, it + g,
                                  [&] { return fragment_key(a.tri_first + t0 + slot, tf.meta, (uint32_t)dxi, (uint32_t)dyi); }, lane);
            __syncwarp();
        }
        __syncthreads();  // the span table and the staged unit may be overwritten from here on
    }
    if (a.world > 1) {  // last CTA out tells every peer that this rank's records have landed
        __threadfence_system();
        __syncthreads();
        if (threadIdx.x == 0) {
            const uint32_t done = atomicAdd(SCHED(a, 6), 1u);
            if (done == gridDim.x - 1) {
                *SCHED(a, 6) = 0;
                __threadfence_system();
                for (uint32_t i = 0; i < a.world; ++i) {
                    const uint32_t p = (a.rank + 1u + i) % a.world;
                    st_release_sys(a.peer_xch[p] + a.rank * 4 + 2, a.epoch);
                }
            }
        }
    }
#ifdef M2S_TRACE
    __syncthreads();   // the end of the step as scripts/trace_raster.py places it: the last CTA's last record written
    if (a.trace && threadIdx.x == 0) atomicMax(a.trace + kTrFragEndNs, gtimer_ns());
#endif
}

// waits until every rank's records of this epoch have landed in THIS rank's final buffer, publishes the
// number of records it holds: the ranks' stored counts summed, cut at the buffer's capacity gcap (emit_records
// clips every span there); one thread — the data path never returns to the host
__global__ void gather_wait_kernel(const unsigned long long* xch, uint32_t world, unsigned long long epoch,
                                   unsigned long long gcap, unsigned long long* total_global, uint32_t* status) {
    unsigned long long tot = 0;
    for (uint32_t r = 0; r < world; ++r) {
        wait_epoch(xch + r * 4 + 2, epoch, status, 2u);
        tot += *reinterpret_cast<const volatile unsigned long long*>(xch + r * 4);
    }
    if (total_global) *total_global = tot < gcap ? tot : gcap;
}

// ------------------------------------------------------------------------------------------
// host side, declared in m2s_device.cuh
// ------------------------------------------------------------------------------------------
// f(std::integral_constant<int, LAYOUT>) for `layout`
template <class F>
static auto with_layout(int layout, F&& f) {
    switch (layout) {
        case 0: return f(std::integral_constant<int, 0>{});
        case 1: return f(std::integral_constant<int, 1>{});
        case 2: return f(std::integral_constant<int, 2>{});
        case 3: return f(std::integral_constant<int, 3>{});
        default: return f(std::integral_constant<int, 4>{});
    }
}

cudaError_t fragment_configure(int layout, int* blocks_per_sm) {
    return with_layout(layout, [&](auto l) {
        cudaError_t e = cudaFuncSetAttribute(fragment_kernel<l>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FragSmem<l>::kBytes);
        if (e != cudaSuccess) return e;
        return cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm, fragment_kernel<l>, kFragThreads, FragSmem<l>::kBytes);
    });
}

cudaError_t fragment_launch(int layout, const ConvertArgs& args, int grid, bool pdl, cudaStream_t stream) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(kFragThreads);
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;  // PDL: overlap this launch with the raster kernel's tail
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl ? 1 : 0;
    return with_layout(layout, [&](auto l) {
        cfg.dynamicSmemBytes = FragSmem<l>::kBytes;
        return cudaLaunchKernelEx(&cfg, fragment_kernel<l>, args);
    });
}

cudaError_t gather_wait_launch(const unsigned long long* xch, uint32_t world, unsigned long long epoch, unsigned long long gcap,
                               unsigned long long* total_global, uint32_t* status, cudaStream_t stream) {
    gather_wait_kernel<<<1, 1, 0, stream>>>(xch, world, epoch, gcap, total_global, status);
    return cudaGetLastError();
}

}  // namespace m2s
