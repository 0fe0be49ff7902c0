// m2s_kernels.cu — the conversion pass as hand-written sm_90a CUDA.
//
// Two kernels on one stream replace the reference's geometry shader, fixed-function rasteriser, fragment shader
// and SSBO atomic append (converter{GS,FS}.glsl, ConversionPass.cpp:114-116).  The second kernel is launched with
// programmatic dependent launch.  What crosses between them is small and stays in the 50 MB L2: one 176-192 B
// record per triangle, 288 B per queued work item — never anything per fragment.
//
// raster_kernel — per-TRIANGLE work: set-up and COUNTING (persistent, one CTA per SM, every warp an autonomous
// pipeline; one __syncthreads after the descriptor tables are copied to shared memory, none in the steady state)
//   work unit = <= 32 consecutive triangles; a warp's first unit is static (global warp id), further ones are
//     claimed from a global counter; the next unit's triangles are in flight (TMA) while this one is processed
//   TMA (cp.async.bulk + mbarrier complete_tx) stages the unit's 144 B/triangle into shared memory
//   per-triangle stage, one LANE per triangle (converterGS.glsl:326-443): longest edge, face normal, dominant
//     axis, orthographic uv, quaternion, UV->3D Jacobian scale; rasteriser set-up: 24.8 fixed-point window
//     coords, int64 edge functions, top-left ownership bits, candidate pixel box (clamped to the call's
//     pixel-row band); the triangle's resolved sampler state (mip level pair, blend fraction, level offsets)
//   coverage is only COUNTED here:
//     small triangles (box <= 64 pixels, <= 32 rows, int32-safe): lane-per-triangle lock-step walk of the box
//       with incremental edge functions -> 64-bit coverage mask, stored in the record; a warp scan gives every
//       triangle its offset inside the unit; ONE global atomicAdd per unit reserves the output range
//       (the reference: one atomicCounterIncrement per fragment)
//     all other triangles: lane-per-ROW exact interval (m2s_span.cuh: three estimated divisions + exact int64
//       fix-up) -> fragments per block of 32 rows; blocks are batched into work items (<= 32 blocks or
//       >= 1024 fragments; one atomicAdd reserves the item's output range), a block of more than 2048
//       fragments is cut into several items — a 2-triangle quad at R = 2048 becomes 4096 items for the
//       whole GPU, while its raster work is 128 warp steps
//   the unit's records leave shared memory as ONE TMA bulk store (cp.async.bulk.global.shared::cta)
//   PACKED56 records also carry the varyings the layout needs (position, uv) as PLANES over the pixel grid (fp64
//     coefficients from the exact edge functions): the fragment stage needs neither the vertices nor 64-bit arithmetic
//   DIRECT path (PACKED56, launches where the warps take several units each): the small triangles of a light unit are
//     shaded by the warp that rasterised them, straight from the records in its shared-memory slice (direct_run)
// fragment_kernel — per-FRAGMENT work (converterFS.glsl:44-104); a CTA of 4 warps takes one work item:
//   TMA stages the unit's records (three-map layouts: and its 144 B/triangle vertices) into shared memory, every
//   warp rebuilds the row spans of its share of the item's blocks (mask rows / m2s_span.cuh) into a prefix
//   table; then a warp takes 32 consecutive fragments = 32 consecutive output records: a search between the group's
//   first and last row gives (triangle, x, y); varyings from the planes (PACKED56) or from the staged vertices with
//   exact barycentrics (REF96, .ply rows); all texel loads of all bound maps issued back to back,
//   trilinear filter on the FMA pipe (u8->f32 by PRMT+FADD), TBN normal, encode (REF96 / PACKED56 / the three
//   .ply row formats directly); the 32 records are transposed through shared memory and written as one
//   contiguous span (16-byte body whatever the alignment of the span) — locally, or into every rank's final buffer
//   over NVLink (fused multi-GPU gather), or after the earlier chunks' records (appended launches of the host path).
//
// Bit-exactness: every float operation of the per-triangle stage is written with __f*_rn intrinsics in the
// operation order of the oracle (and of GLM, which the reference's GLSL-as-C++ build uses): coverage is
// bit-exact and Scale/Quaternion match converterGS.glsl bit for bit.  Per-fragment values may use FMA
// contraction / fast reciprocals and are compared with a tolerance.
#include <cstddef>
#include <cstdio>
#include "m2s_codec.cuh"
#include "m2s_device.cuh"
#include "m2s_span.cuh"

// resident raster warps per SM / register cap per raster kind (warps are a multiple of 4: register allocation granularity)
#ifndef M2S_RASTER_WARPS
#define M2S_RASTER_WARPS 16
#endif
#ifndef M2S_RASTER_WARPS_3MAP
#define M2S_RASTER_WARPS_3MAP 16
#endif
#ifndef M2S_RASTER_REGS
#define M2S_RASTER_REGS 128
#endif
#ifndef M2S_FRAG_WARPS
#define M2S_FRAG_WARPS 4
#endif
#ifndef M2S_FRAG_THREADS_P56
#define M2S_FRAG_THREADS_P56 1024   // resident fragment-kernel threads per SM for PACKED56 (register cap = 65536 / this)
#endif
// (a second staged-unit buffer with the next item's TMA in flight was measured in r02: no gain, it costs a resident CTA
// per SM and the other CTAs already hide the load; removed)

namespace m2s {

// ------------------------------------------------------------------------------------------
// PTX helpers: mbarrier + 1-D bulk async copy (TMA engine; SASS UBLKCP)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tma_store_1d(void* dst_gmem, const void* src_smem, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem), "r"(smem_u32(src_smem)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// M2S_TRACE builds: per-warp SUMS over all the warp's units, 16 slots per raster warp (scripts/trace_raster.py).
// Phases are clock64() deltas (SM cycles: the globaltimer ticks too coarsely for one unit); TR_PHASE adds the cycles
// since the previous mark to its slot.  Fire-and-forget atomics: the trace adds no wait to the chain it measures.
enum TraceSlot {
    kTrLoadWait, kTrSetup, kTrWalkScan, kTrLarger, kTrReserve, kTrList, kTrShade, kTrUnitEnd, kTrTail,
    kTrUnits, kTrDirectUnits, kTrGroups, kTrCycles, kTrNanos, kTrEntry
};
#ifdef M2S_TRACE
__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
#define TR_SLOT(s) (((size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * 16 + (s))
#define TR_PHASE(a, s) do { const long long n_ = clock64(); if ((a).trace && (threadIdx.x & 31) == 0) atomicAdd((a).trace + TR_SLOT(s), (unsigned long long)(n_ - tr_prev_)); tr_prev_ = n_; } while (0)
#define TR_ADD(a, s, v) do { if ((a).trace && (threadIdx.x & 31) == 0) atomicAdd((a).trace + TR_SLOT(s), (unsigned long long)(v)); } while (0)
#else
#define TR_PHASE(a, s) do { } while (0)
#define TR_ADD(a, s, v) do { } while (0)
#endif
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long gtimer_ns() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
// Bounded wait for a peer's flag (fused gather): a rank that never launches its kernels must not hang every GPU of the
// node forever.  After kSpinTimeoutNs the waiter gives up, raises bit `why` in the context's status word (mapped pinned
// host memory, read by m2s_ctx_status) and carries on with whatever it has — the host call then reports M2S_E_CUDA.
constexpr unsigned long long kSpinTimeoutNs = 2000000000ull;
__device__ __forceinline__ bool wait_epoch(const unsigned long long* flag, unsigned long long epoch, uint32_t* status, uint32_t why) {
    if (ld_acquire_sys(flag) == epoch) return true;
    const unsigned long long t0 = gtimer_ns();
    unsigned ns = 100;
    while (ld_acquire_sys(flag) != epoch) {
        __nanosleep(ns);
        ns = min(ns * 2u, 2000u);
        if (gtimer_ns() - t0 > kSpinTimeoutNs) {
            if (status) { *reinterpret_cast<volatile uint32_t*>(status) = why; __threadfence_system(); }  // plain store: zero-copy memory
            return false;
        }
    }
    return true;
}
constexpr int kSchedStride = 32;  // scheduler words live on separate 128-byte lines
#define SCHED(a, i) ((a).sched + (i) * kSchedStride)
__device__ __forceinline__ void prefetch_l2(const void* p, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_u32(const uint32_t* p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// ------------------------------------------------------------------------------------------
// exact fp32 (one rounding per operation, GLM operation order)
// ------------------------------------------------------------------------------------------
struct f3 {
    float x, y, z;
};
__device__ __forceinline__ f3 sub3(f3 a, f3 b) { return {__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y), __fsub_rn(a.z, b.z)}; }
__device__ __forceinline__ f3 scale3(f3 a, float s) { return {__fmul_rn(a.x, s), __fmul_rn(a.y, s), __fmul_rn(a.z, s)}; }
__device__ __forceinline__ float dot3(f3 a, f3 b) {
    return __fadd_rn(__fadd_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)), __fmul_rn(a.z, b.z));
}
__device__ __forceinline__ float len3(f3 a) { return __fsqrt_rn(dot3(a, a)); }
__device__ __forceinline__ f3 norm3(f3 a) { return scale3(a, __fdiv_rn(1.0f, __fsqrt_rn(dot3(a, a)))); }
__device__ __forceinline__ f3 cross3(f3 x, f3 y) {
    return {__fsub_rn(__fmul_rn(x.y, y.z), __fmul_rn(y.y, x.z)), __fsub_rn(__fmul_rn(x.z, y.x), __fmul_rn(y.z, x.x)),
            __fsub_rn(__fmul_rn(x.x, y.y), __fmul_rn(y.x, x.y))};
}

// ------------------------------------------------------------------------------------------
// per-triangle record: everything the fragment kernel needs besides the vertices
// ------------------------------------------------------------------------------------------
struct __align__(8) TexRef {  // 16 B — one map, resolved for one triangle
    uint32_t off0, off1;          // texel offsets of the two mip levels in the arena; off0 == ~0u: no map
    unsigned short w0, h0, w1, h1;
};
// Three-map layouts (REF96, the .ply rows): 176 B — the fragment stage interpolates the varyings from the staged vertices
// with exact barycentrics (12 varyings as planes would make the record 336 B: 16 warp slices of the raster kernel would
// no longer fit in shared memory, and 12 warps per SM need two rounds for the 70 k-triangle bench scene: measured
// 81 vs 62 us).
template <int NMAPS>
struct __align__(16) TriRec {
    // exact barycentrics: lambda_k(x,y) = (E0_k + A_k (x-x0) + B_k (y-y0)) * inv_area  (GL 4.6 eq. 14.9, w = 1);
    // coverage: E0_k - (edge k owns its zero set ? 0 : 1) >= 0
    long long E0[3];              // edge functions at the centre of pixel (x0, y0), the box origin
    unsigned long long hits;      // small triangles: coverage mask of the w x h box, bit = row * w + column
    int A[3];
    int B[3];
    unsigned box;                 // w (13 bits) | h (13) << 13 | ownership bits (3) << 26 | small (1) << 29; 0: nothing to emit
    unsigned meta;                // bits 0-2: map m has the same level sizes as map 0 (=> same footprint and weights);
                                  // bits 4-15: x0, bits 16-27: y0 of the candidate pixel box
    unsigned first;               // small triangles of the unit before this one: their fragments (low 16 bits) and their
                                  // box rows (high 16 bits) — the triangle's place in the unit item's span table
    float inv_area;
    float sx, sy;                 // scale[0..1]: raw (REF96) or log(scale * sigma/R); the third component is a constant
    float frac[NMAPS];            // trilinear blend per map (0 => single level)
    float quat[4];                // (w,x,y,z)
    float factor[4];              // u_materialFactor
    TexRef tex[NMAPS];            // resolved sampler state per map
};
// One map (PACKED56): 192 B — the varyings the layout carries (position, uv) as PLANES over the pixel grid; the fragment
// stage needs neither the vertices nor 64-bit arithmetic.
template <>
struct __align__(16) TriRec<1> {
    long long E0[3];
    unsigned long long hits;
    int A[3];
    int B[3];
    unsigned box;
    unsigned meta;
    unsigned first;
    float frac[1];
    TexRef tex[1];
    float sx;                     // log(scale[0] * sigma/R)
    float pad_;
    float quat[4];                // (w,x,y,z)                                  — 16-byte aligned from here on
    float factor[4];              // u_materialFactor
    // value(x, y) = base + (x-x0) ddx + (y-y0) ddy (affine in window space, GL 4.6 eq. 14.9 with w = 1), stored as
    // {base4, ddx4, ddy4} of (Px, Py, Pz, u), then (v, dv/dx, dv/dy).  Computed once per triangle in fp64 from the exact
    // edge functions
    float plane[15];
    float sy;                     // log(scale[1] * sigma/R); the third component is a constant
};
static_assert(sizeof(TriRec<1>) == 192 && sizeof(TriRec<3>) == 176, "TriRec layout");
static_assert(offsetof(TriRec<1>, quat) % 16 == 0 && offsetof(TriRec<1>, plane) % 16 == 0, "TriRec<1> alignment");
constexpr unsigned kBoxSmall = 1u << 29;

// raster kinds: what the per-triangle stage has to prepare (maps to resolve, raw or log scale)
template <int RK> struct RCfg;
template <> struct RCfg<0> { static constexpr int kMaps = 3, kWarps = M2S_RASTER_WARPS_3MAP; static constexpr bool kLogScale = false; };  // REF96
template <> struct RCfg<1> { static constexpr int kMaps = 1, kWarps = M2S_RASTER_WARPS; static constexpr bool kLogScale = true; };        // PACKED56
template <> struct RCfg<2> { static constexpr int kMaps = 3, kWarps = M2S_RASTER_WARPS_3MAP; static constexpr bool kLogScale = true; };   // .ply rows

// output layouts (m2s_layout)
template <int LAYOUT> struct Cfg;
template <> struct Cfg<0> { static constexpr int kStride = 96, kRK = 0; };   // REF96
template <> struct Cfg<1> { static constexpr int kStride = 56, kRK = 1; };   // PACKED56 (fragment kernel: 8 CTAs/SM = 64 registers)
template <> struct Cfg<2> { static constexpr int kStride = 248, kRK = 2; };  // PLY_STANDARD (parsers.cpp:431-514)
template <> struct Cfg<3> { static constexpr int kStride = 76, kRK = 2; };   // PLY_PBR      (parsers.cpp:232-316)
template <> struct Cfg<4> { static constexpr int kStride = 48, kRK = 2; };   // PLY_COMPRESSED (parsers.cpp:339-428)

template <int RK>
struct __align__(128) WarpBlock {
    float4 tri[kUnitTris * 9];                    // 4608 B, TMA destination
    TriRec<RCfg<RK>::kMaps> rec[kUnitTris];       // TMA source
    BlockRef pend[kStashItems * kItemBlocks];     // the stash: row blocks of up to kStashItems work items
    uint32_t itN[kStashItems];                    // blocks per item | kItUnit / kItSplit
    uint32_t itTotal[kStashItems];                // fragments per item
    uint64_t bar;
};

// The scene's descriptor tables as the set-up sees them: in shared memory when they fit (each CTA copies
// them once — ~2100 warps (132 SMs x 16) chasing range -> primitive -> texture through the same few L2 lines pay a
// contended L2 round trip per dependent step), else in global memory.
struct Tables {
    const DRange* ranges;
    const DPrim* prims;
    const DTexture* texs;
    uint32_t nranges;
};
constexpr uint32_t kTableSmemBytes = 16 * 1024;

// what the raster kernel itself keeps of a triangle after the set-up (registers of the owning lane)
struct TriSetup {
    long long E0[3];
    int A[3], B[3];
    int w, h;
    unsigned incl;
};

// ------------------------------------------------------------------------------------------
// per-triangle stage + rasteriser set-up.  t4: 9 float4 in shared memory.
// Returns the number of candidate pixels (0 => nothing to rasterise).
// ------------------------------------------------------------------------------------------
template <int RK>
__device__ __forceinline__ uint32_t setup_triangle(const float4* __restrict__ t4, uint32_t tri_global, const ConvertArgs& a,
                                                   const Tables& tb, TriSetup& ts, TriRec<RCfg<RK>::kMaps>& tf) {
    using C = RCfg<RK>;
    // triangle -> primitive (sorted disjoint ranges)
    int lo = 0, hi = (int)tb.nranges - 1, found = -1;
    while (lo <= hi) {
        const int mid = (lo + hi) >> 1;
        const DRange r = tb.ranges[mid];
        if (tri_global < r.first) hi = mid - 1;
        else if (tri_global >= r.end) lo = mid + 1;
        else { found = (int)r.prim; break; }
    }
    if (found < 0) return 0;
    const DPrim pr = tb.prims[found];

    // vertex data: 3 x {pos3 nrm3 tan4 uv2} = 9 float4
    const float4 q0 = t4[0], q3 = t4[3], q6 = t4[6];
    const float4 q2 = t4[2], q5 = t4[5], q8 = t4[8];
    const f3 P0 = {q0.x, q0.y, q0.z}, P1 = {q3.x, q3.y, q3.z}, P2 = {q6.x, q6.y, q6.z};

    // converterGS.glsl:327-347
    f3 e1 = sub3(P1, P0), e2 = sub3(P2, P0), e3 = sub3(P2, P1);
    const float l1 = len3(e1), l2 = len3(e2), l3 = len3(e3);
    if (l2 > l1 && l2 > l3) { f3 tmp = e1; e1 = e2; e2 = tmp; }
    else if (l3 > l1 && l3 > l2) { e1 = e3; }
    e1 = norm3(e1);
    const f3 n = norm3(cross3(e1, e2));
    const float ax = fabsf(n.x), ay = fabsf(n.y), az = fabsf(n.z);
    const int axis = (ax > ay && ax > az) ? 0 : ((ay > az) ? 1 : 2);

    // :354-397 orthogonal uv: X -> (y,z), Y -> (x,z), Z -> (x,y), over max(range_a, range_b)
    float ou[3], ov[3];
    {
        const float mina = axis == 0 ? pr.bmin[1] : pr.bmin[0], maxa = axis == 0 ? pr.bmax[1] : pr.bmax[0];
        const float minb = axis == 2 ? pr.bmin[1] : pr.bmin[2], maxb = axis == 2 ? pr.bmax[1] : pr.bmax[2];
        const float ra = __fsub_rn(maxa, mina), rb = __fsub_rn(maxb, minb);
        const float range = (ra < rb) ? rb : ra;
        const float pa0 = axis == 0 ? P0.y : P0.x, pa1 = axis == 0 ? P1.y : P1.x, pa2 = axis == 0 ? P2.y : P2.x;
        const float pb0 = axis == 2 ? P0.y : P0.z, pb1 = axis == 2 ? P1.y : P1.z, pb2 = axis == 2 ? P2.y : P2.z;
        ou[0] = __fdiv_rn(__fsub_rn(pa0, mina), range); ov[0] = __fdiv_rn(__fsub_rn(pb0, minb), range);
        ou[1] = __fdiv_rn(__fsub_rn(pa1, mina), range); ov[1] = __fdiv_rn(__fsub_rn(pb1, minb), range);
        ou[2] = __fdiv_rn(__fsub_rn(pa2, mina), range); ov[2] = __fdiv_rn(__fsub_rn(pb2, minb), range);
    }

    // rasteriser set-up first: gl_Position = ouv*2-1 (:439), viewport R x R, 8 sub-pixel bits.  A triangle that
    // cannot emit a fragment leaves here, before the quaternion / Jacobian / sampler arithmetic
    int X[3], Y[3];
    bool valid = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float ndx = __fsub_rn(__fmul_rn(ou[k], 2.0f), 1.0f), ndy = __fsub_rn(__fmul_rn(ov[k], 2.0f), 1.0f);
        const float xw = __fadd_rn(__fmul_rn(ndx, a.half_R), a.half_R), yw = __fadd_rn(__fmul_rn(ndy, a.half_R), a.half_R);
        if (!(fabsf(xw) <= kGuard) || !(fabsf(yw) <= kGuard)) valid = false;  // also rejects NaN
        X[k] = __float2int_rn(__fmul_rn(xw, 256.0f));
        Y[k] = __float2int_rn(__fmul_rn(yw, 256.0f));
    }
    if (!valid) return 0;
    const long long area2 = (long long)(X[1] - X[0]) * (Y[2] - Y[0]) - (long long)(X[2] - X[0]) * (Y[1] - Y[0]);
    if (area2 == 0) return 0;
    const int xmin = min(X[0], min(X[1], X[2])), xmax = max(X[0], max(X[1], X[2]));
    const int ymin = min(Y[0], min(Y[1], Y[2])), ymax = max(Y[0], max(Y[1], Y[2]));
    const int R1 = (int)a.R - 1;
    const int x0 = max(0, (xmin + 127) >> 8), x1 = min(R1, (xmax - 128) >> 8);
    const int y0 = max((int)a.row_begin, (ymin + 127) >> 8), y1 = min((int)a.row_end - 1, (ymax - 128) >> 8);  // row band
    if (x1 < x0 || y1 < y0) return 0;
    const int sg = area2 < 0 ? -1 : 1;
    unsigned incl = 0;
    const float ia = 1.0f / __ll2float_rn(area2 < 0 ? -area2 : area2);
    // edge functions E_k(i,j) = A_k i + B_k j + C_k at pixel centres, sign-normalised; kept relative to the box
    // origin; the per-pixel steps of the mesh uv (constant per triangle: uv is affine in window space)
    float dudx = 0.f, dvdx = 0.f, dudy = 0.f, dvdy = 0.f;
    {
        const float uvx[3] = {q2.z, q5.z, q8.z}, uvy[3] = {q2.w, q5.w, q8.w};
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const int va = (k + 1) % 3, vb = (k + 2) % 3;
            const int dx = X[vb] - X[va], dy = Y[vb] - Y[va];
            const int A = sg * (-dy * 256), B = sg * (dx * 256);
            const long long Ck = (long long)sg * ((long long)dx * (128 - Y[va]) - (long long)dy * (128 - X[va]));
            if (A > 0 || (A == 0 && B > 0)) incl |= 1u << k;
            const long long E0 = Ck + (long long)A * x0 + (long long)B * y0;
            ts.E0[k] = E0; ts.A[k] = A; ts.B[k] = B;
            tf.E0[k] = E0; tf.A[k] = A; tf.B[k] = B;
            const float ca = (float)A * ia, cb = (float)B * ia;
            dudx += uvx[k] * ca; dvdx += uvy[k] * ca;
            dudy += uvx[k] * cb; dvdy += uvy[k] * cb;
        }
    }
    ts.incl = incl;
    ts.w = x1 - x0 + 1; ts.h = y1 - y0 + 1;
    if constexpr (C::kMaps != 1) tf.inv_area = ia;
    // one map: the varyings as planes over the pixel grid.  lambda_k(x, y) = (E0_k + A_k (x-x0) + B_k (y-y0)) / |area2| belongs to
    // vertex k; base / ddx / ddy of a varying are the lambda-weighted sums of its three vertex values.  fp64: for a thin
    // triangle the box origin lies far outside it and |lambda| >> 1 — the sums cancel (an fp32 version put 5e-4 of error
    // into positions of the golden-vector triangles); the correctly rounded coefficients themselves are benign (the
    // varyings are affine over the whole box), so a fragment's value is two fp32 FMAs away from the exact interpolation
#ifndef M2S_EXP_NOPLANES   // timing experiment only: no planes (wrong output)
    if constexpr (C::kMaps == 1) {
        const double inv = 1.0 / (double)(area2 < 0 ? -area2 : area2);
        const double lb0 = (double)ts.E0[0] * inv, lb1 = (double)ts.E0[1] * inv, lb2 = (double)ts.E0[2] * inv;
        const double lx0 = (double)ts.A[0] * inv, lx1 = (double)ts.A[1] * inv, lx2 = (double)ts.A[2] * inv;
        const double ly0 = (double)ts.B[0] * inv, ly1 = (double)ts.B[1] * inv, ly2 = (double)ts.B[2] * inv;
        auto put = [&](int at, int stride, float v0, float v1, float v2) {  // base at plane[at], ddx at [at + stride], ddy at [at + 2 stride]
            const double a0 = (double)v0, a1 = (double)v1, a2 = (double)v2;
            tf.plane[at] = (float)(lb0 * a0 + lb1 * a1 + lb2 * a2);
            tf.plane[at + stride] = (float)(lx0 * a0 + lx1 * a1 + lx2 * a2);
            tf.plane[at + 2 * stride] = (float)(ly0 * a0 + ly1 * a1 + ly2 * a2);
        };
        put(0, 4, q0.x, q3.x, q6.x); put(1, 4, q0.y, q3.y, q6.y); put(2, 4, q0.z, q3.z, q6.z);   // position
        put(3, 4, q2.z, q5.z, q8.z);                                                             // u
        put(12, 1, q2.w, q5.w, q8.w);                                                            // v
    }
#endif

    // :399-407 rotation -> quaternion (w,x,y,z), quat_cast :131-183
    {
        const f3 xA = e1, yA = norm3(cross3(n, xA)), zA = n;
        const float m00 = xA.x, m01 = xA.y, m02 = xA.z, m10 = yA.x, m11 = yA.y, m12 = yA.z, m20 = zA.x, m21 = zA.y,
                    m22 = zA.z;
        const float fX = __fsub_rn(__fsub_rn(m00, m11), m22), fY = __fsub_rn(__fsub_rn(m11, m00), m22),
                    fZ = __fsub_rn(__fsub_rn(m22, m00), m11), fW = __fadd_rn(__fadd_rn(m00, m11), m22);
        int big = 0;
        float fB = fW;
        if (fX > fB) { fB = fX; big = 1; }
        if (fY > fB) { fB = fY; big = 2; }
        if (fZ > fB) { fB = fZ; big = 3; }
        const float bv = __fmul_rn(__fsqrt_rn(__fadd_rn(fB, 1.0f)), 0.5f);
        const float mult = __fdiv_rn(0.25f, bv);
        float w, x, y, z;
        if (big == 0) { w = bv; x = __fmul_rn(__fsub_rn(m12, m21), mult); y = __fmul_rn(__fsub_rn(m20, m02), mult); z = __fmul_rn(__fsub_rn(m01, m10), mult); }
        else if (big == 1) { w = __fmul_rn(__fsub_rn(m12, m21), mult); x = bv; y = __fmul_rn(__fadd_rn(m01, m10), mult); z = __fmul_rn(__fadd_rn(m20, m02), mult); }
        else if (big == 2) { w = __fmul_rn(__fsub_rn(m20, m02), mult); x = __fmul_rn(__fadd_rn(m01, m10), mult); y = bv; z = __fmul_rn(__fadd_rn(m12, m21), mult); }
        else { w = __fmul_rn(__fsub_rn(m01, m10), mult); x = __fmul_rn(__fadd_rn(m20, m02), mult); y = __fmul_rn(__fadd_rn(m12, m21), mult); z = bv; }
        tf.quat[0] = w; tf.quat[1] = x; tf.quat[2] = y; tf.quat[3] = z;
    }

    // :269-300,206-235,414-430 Jacobian scale
    {
        const float ja = __fsub_rn(ou[1], ou[0]), jb = __fsub_rn(ou[2], ou[0]);
        const float jc = __fsub_rn(ov[1], ov[0]), jd = __fsub_rn(ov[2], ov[0]);
        const float det = __fsub_rn(__fmul_rn(ja, jd), __fmul_rn(jc, jb));
        float i00 = 0.f, i10 = 0.f, i01 = 0.f, i11 = 0.f;
        if (det != 0.0f) {
            const float invDet = __fdiv_rn(1.0f, det);
            i00 = __fmul_rn(jd, invDet); i10 = __fmul_rn(-jb, invDet); i01 = __fmul_rn(-jc, invDet); i11 = __fmul_rn(ja, invDet);
        }
        const f3 V0 = sub3(P1, P0), V1 = sub3(P2, P0);
        const f3 Ju = {__fadd_rn(__fmul_rn(V0.x, i00), __fmul_rn(V1.x, i01)), __fadd_rn(__fmul_rn(V0.y, i00), __fmul_rn(V1.y, i01)),
                       __fadd_rn(__fmul_rn(V0.z, i00), __fmul_rn(V1.z, i01))};
        const f3 Jv = {__fadd_rn(__fmul_rn(V0.x, i10), __fmul_rn(V1.x, i11)), __fadd_rn(__fmul_rn(V0.y, i10), __fmul_rn(V1.y, i11)),
                       __fadd_rn(__fmul_rn(V0.z, i10), __fmul_rn(V1.z, i11))};
        // Scale and Quaternion are bit-identical to converterGS.glsl's (tests: golden GS vectors), and so is the log
        // of the packed / .ply layouts (glibc's logf, m2s_codec.cuh)
        const float sx = len3(Ju), sy = len3(Jv);
        if (C::kLogScale) {  // parsers.cpp:497-499 log(scale * sigma/R)
            tf.sx = log_scale(sx, a.mult); tf.sy = log_scale(sy, a.mult);
        } else { tf.sx = sx; tf.sy = sy; }
    }
    tf.factor[0] = pr.factor[0]; tf.factor[1] = pr.factor[1]; tf.factor[2] = pr.factor[2]; tf.factor[3] = pr.factor[3];

    // sampler state (GL 4.6 8.14): the steps of the mesh uv are constant per triangle, so lambda, the
    // level pair and the blend fraction are too
    unsigned share = 0;
    TexRef ref0;
    float frac0 = 0.f;
#pragma unroll
    for (int m = 0; m < C::kMaps; ++m) {
        TexRef ref;
        ref.off0 = 0xffffffffu; ref.off1 = 0; ref.w0 = ref.h0 = ref.w1 = ref.h1 = 1;
        float frac = 0.f;
        const int ti = pr.tex[m];
        if (ti >= 0) {
            const DTexture& t = tb.texs[ti];  // indexed in place (a local copy indexed by level would live in local memory)
            const float W = (float)t.w[0], H = (float)t.h[0];
            const float axx = dudx * W, bxx = dvdx * H, ayy = dudy * W, byy = dvdy * H;
            const float lam = 0.5f * __log2f(fmaxf(axx * axx + bxx * bxx, ayy * ayy + byy * byy));  // log2 of the longer step
            const int q = (int)t.nlevels - 1;
            int l0 = 0;
            if (!(lam > 0.0f)) { l0 = 0; }                       // magnification: LINEAR on level 0
            else if (lam >= (float)q) { l0 = q; }                 // clamped to the last level
            else { const float d = floorf(lam); l0 = (int)d; frac = lam - d; }
            const int l1 = min(l0 + 1, q);
            ref.off0 = t.off[l0]; ref.off1 = t.off[l1];
            ref.w0 = t.w[l0]; ref.h0 = t.h[l0]; ref.w1 = t.w[l1]; ref.h1 = t.h[l1];
        }
        if (m == 0) { ref0 = ref; frac0 = frac; }
        else if (ti >= 0 && ref0.off0 != 0xffffffffu && ref.w0 == ref0.w0 && ref.h0 == ref0.h0 && ref.w1 == ref0.w1 &&
                 ref.h1 == ref0.h1 && frac == frac0)
            share |= 1u << m;
        tf.tex[m] = ref;
        tf.frac[m] = frac;
    }
    tf.meta = share | ((unsigned)x0 << 4) | ((unsigned)y0 << 16);
    return (uint32_t)ts.w * (uint32_t)ts.h;
}

// ------------------------------------------------------------------------------------------
// sampler: RGBA8 unorm, REPEAT, bilinear within a level, linear between levels
// ------------------------------------------------------------------------------------------
// The two mip levels of a trilinear lookup are the two halves of every pair below — .x = level 0, .y = level 1.
// sm_90 has no packed fp32 instructions: a pair operation is two scalar FMA-pipe instructions, each rounded to
// nearest and never contracted, so every lane computes exactly what the scalar oracle order prescribes.
__device__ __forceinline__ float2 f2(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ float2 f2(float a) { return make_float2(a, a); }
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
struct Bilin2 {             // the 2x2 footprints of one map on its two mip levels
    uint32_t i00[2], i10[2], i01[2], i11[2];  // texel indices relative to the level starts
    float2 w00, w10, w01, w11;                // weights: bilinear x 1/255 x level blend (1-f, f)
};
// small non-negative int -> float on the FMA pipe (no I2F): 2^23 | v is the float 2^23 + v
__device__ __forceinline__ float u2f(uint32_t v) { return __uint_as_float(0x4B000000u | v) - 8388608.0f; }
// floor for |x| < 2^22 on the FMA pipe: round-to-nearest of x - 0.5 via the 1.5*2^23 trick.  At exact
// integers it may return x - 1 with fraction 1, which selects the same texels with the same weights.
__device__ __forceinline__ float fast_floor(float x, int& i) {
    const float t = (x - 0.5f) + 12582912.0f;
    i = __float_as_int(t) - 0x4B400000;
    return t - 12582912.0f;
}
__device__ __forceinline__ float2 fast_floor2(float2 x, int& i0, int& i1) {
    const float2 t = fadd2(fadd2(x, f2(-0.5f)), f2(12582912.0f));
    i0 = __float_as_int(t.x) - 0x4B400000;
    i1 = __float_as_int(t.y) - 0x4B400000;
    return fadd2(t, f2(-12582912.0f));
}
// REPEAT in the normalised domain: uv -> [0, 1]; NaN / huge values are pinned first so that the texel indices below
// can never leave the level (fmaxf(NaN, x) = x)
__device__ __forceinline__ float wrap01(float u) {
    int d;
    u = fminf(fmaxf(u, -1048576.0f), 1048576.0f);
    return u - fast_floor(u, d);
}
// the four texel indices of a footprint whose lower-left texel is (ix, iy), ix in [-1, W-1], iy in [-1, H-1]
__device__ __forceinline__ void footprint(int ix, int iy, int W, int H, uint32_t& i00, uint32_t& i10, uint32_t& i01, uint32_t& i11) {
    const int x0 = ix + ((ix >> 31) & W), y0 = iy + ((iy >> 31) & H);   // -1 wraps to the last texel
    const int x1 = x0 + 1 == W ? 0 : x0 + 1, y1 = y0 + 1 == H ? 0 : y0 + 1;
    i00 = (uint32_t)(y0 * W + x0); i10 = (uint32_t)(y0 * W + x1);
    i01 = (uint32_t)(y1 * W + x0); i11 = (uint32_t)(y1 * W + x1);
}
// u, v already wrapped to [0, 1]; lw = level weights (1-f, f) (or (1, 0) for a single level)
__device__ __forceinline__ Bilin2 bilin_setup2(const TexRef& r, float u, float v, float2 lw) {
    const float2 W = f2(u2f(r.w0), u2f(r.w1)), H = f2(u2f(r.h0), u2f(r.h1));
    const float2 x = ffma2(f2(u), W, f2(-0.5f)), y = ffma2(f2(v), H, f2(-0.5f));
    int ix0, ix1, iy0, iy1;
    const float2 fx = fast_floor2(x, ix0, ix1), fy = fast_floor2(y, iy0, iy1);
    const float2 ax = ffma2(fx, f2(-1.0f), x), ay = ffma2(fy, f2(-1.0f), y);
    Bilin2 b;
    footprint(ix0, iy0, (int)r.w0, (int)r.h0, b.i00[0], b.i10[0], b.i01[0], b.i11[0]);
    footprint(ix1, iy1, (int)r.w1, (int)r.h1, b.i00[1], b.i10[1], b.i01[1], b.i11[1]);
    const float2 k = fmul2(lw, f2(1.0f / 255.0f));
    const float2 bx = ffma2(ax, f2(-1.0f), f2(1.0f));
    const float2 cy = fmul2(ay, k), by = ffma2(ay, f2(-k.x, -k.y), k);
    b.w00 = fmul2(bx, by); b.w10 = fmul2(ax, by); b.w01 = fmul2(bx, cy); b.w11 = fmul2(ax, cy);
    return b;
}
// channel CH of the texel pair (level 0, level 1) as floats, without the conversion pipe: 0x4B000000 | byte = 2^23 + byte.
// PRMT takes ONE immediate: with 0x4B000000 as the immediate the selector would need a register (re-materialised per
// use: ~34 extra moves per fragment in the SASS); so the constant lives in a register the compiler cannot fold (k4b,
// produced once per kernel by an opaque mov) and the selector is the immediate.
__device__ __forceinline__ uint32_t opaque_4b() { uint32_t k; asm volatile("mov.u32 %0, 0x4B000000;" : "=r"(k)); return k; }
template <int CH>
__device__ __forceinline__ float2 tex_ch2(uint32_t t0, uint32_t t1, uint32_t k4b) {
    uint32_t a, b;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(a) : "r"(t0), "r"(k4b), "n"(0x7440 | CH));
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(b) : "r"(t1), "r"(k4b), "n"(0x7440 | CH));
    return fadd2(f2(__uint_as_float(a), __uint_as_float(b)), f2(-8388608.0f));
}
// trilinear value of channel CH: tx[0..3] = level-0 texels (00, 10, 01, 11), tx[4..7] = level-1 texels
template <int CH>
__device__ __forceinline__ float filt2(const Bilin2& b, const uint32_t* tx, uint32_t k4b) {
    float2 acc = fmul2(b.w00, tex_ch2<CH>(tx[0], tx[4], k4b));
    acc = ffma2(b.w10, tex_ch2<CH>(tx[1], tx[5], k4b), acc);
    acc = ffma2(b.w01, tex_ch2<CH>(tx[2], tx[6], k4b), acc);
    acc = ffma2(b.w11, tex_ch2<CH>(tx[3], tx[7], k4b), acc);
    return acc.x + acc.y;
}

// ------------------------------------------------------------------------------------------
// raster_kernel helpers: work items of the fragment kernel
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t block_ref(uint32_t slot, uint32_t row_begin, uint32_t nrows) {
    return slot | (row_begin << 5) | (nrows << 17);
}

// A warp collects the work items of its current unit in shared memory (WarpBlock::pend / it*) and publishes them
// with ONE 64-bit atomicAdd that reserves both the output range (low 40 bits: fragments) and the queue slots
// (high 24 bits) — the reference does one atomicCounterIncrement per fragment (converterFS.glsl:46).
struct Stash {            // warp-uniform registers
    uint32_t n_it;        // closed items
    uint32_t cur_nb;      // blocks of the open item
    uint32_t cur_total;   // fragments of the open item
    uint32_t frags;       // fragments of the closed items
    uint32_t slots;       // queue slots of the closed items
    unsigned long long seen;  // a lower bound of the global fragment counter (from this warp's last reservation)
};
constexpr uint32_t kItUnit = 0x80000000u;   // item = the unit's small triangles (one implicit block per triangle)
constexpr uint32_t kItSplit = 0x40000000u;  // item = one oversized row block, cut into several queue slots
constexpr uint32_t kItMicro = 0x20000000u;  // unit item of <= 32 fragments: the block area holds the fragments themselves
                                            // (slot | x << 5 | y << 11, box-relative), one warp shades it with direct loads

template <int RK>
// `extra`: fragments the warp shades itself (direct path) — reserved with the same atomic, after the items' fragments; returns
// the output index of the first of them
__device__ __forceinline__ unsigned long long stash_flush(const ConvertArgs& a, WarpBlock<RK>& wb, uint32_t unit, Stash& st, int lane, uint32_t extra = 0) {
    if (st.n_it == 0 && extra == 0) return 0ull;
    __syncwarp();  // lane 0's stash writes are visible to the warp
    // converterFS.glsl:48-51: the counter keeps counting, but once this warp has SEEN the counter beyond the cap its
    // items cannot emit anything and take no queue slots (at most one reservation per warp straddles the cap; the
    // host sizes the queue for that)
    const uint32_t want = st.seen < a.cap ? st.slots : 0u;
    unsigned long long r = 0;
    if (lane == 0) r = atomicAdd(a.counter, ((unsigned long long)want << 40) | (unsigned long long)(st.frags + extra));
    r = __shfl_sync(0xffffffffu, r, 0);
    const unsigned long long base = r & kFragMask;
    uint32_t slot = (uint32_t)(r >> 40);
    st.seen = base + st.frags + extra;
    const unsigned long long extra_first = base + st.frags;
    if (want) {
        unsigned long long first = base;
        for (uint32_t i = 0; i < st.n_it; ++i) {
            const uint32_t nb = wb.itN[i], tot = wb.itTotal[i];
            const BlockRef* blk = wb.pend + i * kItemBlocks;
            if (nb & kItSplit) {  // fragments [k * item_max, ...) of the one block per slot
                const uint32_t nit = (tot + a.item_max_frags - 1) / a.item_max_frags;
                for (uint32_t k = lane; k < nit; k += 32) {
                    if (slot + k >= a.queue_cap) break;
                    FragItem* it = a.items + slot + k;
                    const uint32_t fb = k * a.item_max_frags;
                    *reinterpret_cast<uint4*>(it) = make_uint4((uint32_t)first, (uint32_t)(first >> 32), unit, 1u);
                    *(reinterpret_cast<uint2*>(it) + 2) = make_uint2(fb, min(tot, fb + a.item_max_frags));
                    it->blocks[0] = blk[0];
                }
                slot += nit;
            } else {
                if (slot < a.queue_cap) {
                    FragItem* it = a.items + slot;
                    if (lane == 0) {
                        *reinterpret_cast<uint4*>(it) = make_uint4((uint32_t)first, (uint32_t)(first >> 32), unit, nb);
                        *(reinterpret_cast<uint2*>(it) + 2) = make_uint2(0u, tot);
                    }
                    if (nb & kItMicro) { if (lane < 16) it->blocks[lane] = blk[lane]; }   // 32 packed fragments
                    else if (!(nb & kItUnit) && (uint32_t)lane < nb) it->blocks[lane] = blk[lane];
                }
                slot += 1;
            }
            first += tot;
        }
    }
    __syncwarp();
    st.n_it = 0; st.frags = 0; st.slots = 0;
    return extra_first;
}

template <int RK>
__device__ __forceinline__ void stash_close_item(const ConvertArgs& a, WarpBlock<RK>& wb, uint32_t unit, Stash& st, int lane) {
    if (st.cur_nb == 0) return;
    if (lane == 0) { wb.itN[st.n_it] = st.cur_nb; wb.itTotal[st.n_it] = st.cur_total; }
    st.frags += st.cur_total; st.slots += 1; st.n_it += 1;
    st.cur_nb = 0; st.cur_total = 0;
    if (st.n_it == kStashItems) stash_flush<RK>(a, wb, unit, st, lane);
}

// a row block of triangle `slot` holding `bt` fragments
template <int RK>
__device__ __forceinline__ void stash_block(const ConvertArgs& a, WarpBlock<RK>& wb, uint32_t unit, Stash& st,
                                            uint32_t slot, uint32_t row_begin, uint32_t nrows, uint32_t bt, int lane) {
    const uint32_t ref = block_ref(slot, row_begin, nrows);
    if (bt > a.item_max_frags) {  // a block of a huge triangle: several queue slots, each a fragment sub-range of the block
        stash_close_item<RK>(a, wb, unit, st, lane);
        if (lane == 0) {
            wb.itN[st.n_it] = 1u | kItSplit; wb.itTotal[st.n_it] = bt;
            wb.pend[st.n_it * kItemBlocks].prefix = 0; wb.pend[st.n_it * kItemBlocks].ref = ref;
        }
        st.frags += bt; st.slots += (bt + a.item_max_frags - 1) / a.item_max_frags; st.n_it += 1;
        // a reservation takes at most 2 * kMaxSplit queue slots (bounds the slack the host adds to the queue)
        if (st.n_it == kStashItems || st.slots >= kMaxSplit) stash_flush<RK>(a, wb, unit, st, lane);
        return;
    }
    if (lane == 0) {
        BlockRef& b = wb.pend[st.n_it * kItemBlocks + st.cur_nb];
        b.prefix = st.cur_total; b.ref = ref;
    }
    st.cur_nb += 1;
    st.cur_total += bt;
    if (st.cur_nb == kItemBlocks || st.cur_total >= a.flush_frags) stash_close_item<RK>(a, wb, unit, st, lane);
}

// the unit's small triangles as one item (blocks implicit: one per triangle, TriRec::first/hits).  A unit with at
// most 32 such fragments (sub-pixel meshes: most units of a 1 M-triangle scan) lists them in the item instead: the
// fragment kernel then needs neither the staged unit nor its span table.  hits/w/first: this lane's triangle.
template <int RK>
__device__ __forceinline__ void stash_unit_item(const ConvertArgs& a, WarpBlock<RK>& wb, uint32_t unit, Stash& st, uint32_t total_small,
                                                uint32_t ntri, unsigned long long hits, uint32_t w, uint32_t first, int lane) {
    if (total_small == 0) return;
    // the open item (if any) stays open: closed items occupy the slots below n_it, the open one is written at n_it
    // only when it closes — so insert the unit item by closing the open one first
    stash_close_item<RK>(a, wb, unit, st, lane);
    const bool micro = total_small <= 32;
    if (micro) {
        uint32_t* list = reinterpret_cast<uint32_t*>(wb.pend + st.n_it * kItemBlocks);
        const uint32_t inv = (65536u + w - 1u) / w;  // row = bit / w by a 16.16 reciprocal (exact for bit < 64, w <= 64)
        uint32_t k = first;
        while (hits) {
            const uint32_t b = (uint32_t)__ffsll((long long)hits) - 1u;
            hits &= hits - 1ull;
            const uint32_t row = (b * inv) >> 16, col = b - row * w;
            list[k++] = (uint32_t)lane | (col << 5) | (row << 11);
        }
    }
    if (lane == 0) { wb.itN[st.n_it] = ntri | kItUnit | (micro ? kItMicro : 0u); wb.itTotal[st.n_it] = total_small; }
    st.frags += total_small; st.slots += 1; st.n_it += 1;
    if (st.n_it == kStashItems) stash_flush<RK>(a, wb, unit, st, lane);
}

// count the row blocks [rb0, rb1) (32 rows each) of one larger triangle: one lane per pixel row, exact intervals
template <int RK>
__device__ __forceinline__ void count_blocks(const ConvertArgs& a, WarpBlock<RK>& wb, uint32_t unit, Stash& st, const RowState& rs, int h,
                                             uint32_t slot, int rb0, int rb1, int lane) {
    for (int rb = rb0 * 32; rb < h && rb < rb1 * 32; rb += 32) {
        const int yrel = rb + lane;
        int xl;
        const uint32_t n = yrel < h ? span_row(rs, yrel, xl) : 0u;
        const uint32_t bt = __reduce_add_sync(0xffffffffu, n);
        if (bt) stash_block<RK>(a, wb, unit, st, slot, (uint32_t)rb, (uint32_t)min(32, h - rb), bt, lane);
    }
}
template <class RecT>
__device__ __forceinline__ RowState row_state(const RecT& r, int& h) {
    const unsigned box = r.box;
    RowState rs;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        rs.E[k] = r.E0[k] - (((box >> (26 + k)) & 1u) ? 0 : 1);
        rs.A[k] = r.A[k]; rs.B[k] = r.B[k];
    }
    rs.w = (int)(box & 0x1fffu);
    h = (int)((box >> 13) & 0x1fffu);
    return rs;
}

// CTA-local help queue (shared memory): a work unit whose larger triangles add up to many row blocks (a wall of a
// building: 28 triangles x 4 blocks x 2000 fragments) would keep ONE warp busy for hundreds of microseconds while the
// others are done: it posts its tall triangles here, in pieces of kDeferBlocks row blocks, and every warp of the CTA that
// has run out of units takes tickets.  Shared-memory atomics only: a grid-wide queue was tried (r02) and lost to the
// serialisation of same-address global atomics (one per unit / per claim: 8-30 us at 2-30 k units).
struct CtaEntry {
    RowState rs;                  // 64 B
    int h;
    uint32_t unit, slot, rb0, rb1;
    volatile uint32_t ready;      // written last
    uint32_t pad[2];
};
constexpr uint32_t kCtaQueueCap = 40;
struct CtaQueue {
    uint32_t tail;                // entries posted (may exceed the capacity: the poster keeps the overflow)
    uint32_t head;                // tickets taken
    uint32_t active;              // warps of the CTA still inside their unit loop
    uint32_t pad;
    CtaEntry q[kCtaQueueCap];
};

// ------------------------------------------------------------------------------------------
// raster_kernel
// ------------------------------------------------------------------------------------------
// defined below, with the fragment kernel; the raster kernel shades the small triangles of light units itself
template <int LAYOUT>
__device__ __forceinline__ void shade(const ConvertArgs& a, const TriRec<RCfg<Cfg<LAYOUT>::kRK>::kMaps>& tf, const float4* __restrict__ v,
                                      int dxi, int dyi, const uint32_t* __restrict__ texb, unsigned char* __restrict__ srec_bytes);
template <int STRIDE>
__device__ __forceinline__ void copy_span(uint8_t* dstbase, unsigned long long boff, const unsigned char* stage, uint32_t nbytes, int lane);
template <int STRIDE>
__device__ __forceinline__ uint32_t stage_shift(unsigned long long record_index);
// DIRECT path: the fragments of a light unit's small triangles, listed in the unit's shared-memory slice, are shaded
// by the warp that rasterised them, in groups of 32 (direct_run).  Used when the warps have several units each
// (n_units > resident warps: on an H100 (132 SMs x 16 warps x 32 triangles) meshes of > 67 k triangles, where most units emit a handful of fragments and a work item
// + a staged unit per unit would cost more than the shading); with one unit per warp the 16 warps of an SM are too
// few to hide the latency of the shading chain and the unit goes to the fragment kernel (that was faster than the direct path,
// also with CTA-level group stealing and software pipelining, when measured during development).
template <int RK>
__device__ __noinline__ void direct_run(const ConvertArgs& a, WarpBlock<RK>& wb, uint32_t total, unsigned long long dfirst, uint32_t t0,
                                        unsigned long long base_prev, unsigned long long room, int lane);

template <int RK>
__global__ void __launch_bounds__(RCfg<RK>::kWarps * 32, 1) raster_kernel(const __grid_constant__ ConvertArgs a) {
    using C = RCfg<RK>;
    using Rec = TriRec<C::kMaps>;
    extern __shared__ __align__(128) unsigned char smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    WarpBlock<RK>& wb = *reinterpret_cast<WarpBlock<RK>*>(smem + (size_t)warp * sizeof(WarpBlock<RK>));
    const unsigned char* tri_bytes = reinterpret_cast<const unsigned char*>(a.tris);
#ifdef M2S_TRACE
    long long tr_prev_ = clock64();
    const long long tr_c0_ = tr_prev_;
    const unsigned long long tr_ns0_ = gtime();
#endif

#ifdef M2S_EARLY_TRIGGER
    // PDL early trigger: one fragment-kernel CTA per SM becomes resident beside this CTA (37 KB of shared memory are
    // left) and parks in griddepcontrol.wait; it starts the moment this grid has drained instead of being launched then
    asm volatile("griddepcontrol.launch_dependents;");
#endif
    if (lane == 0) {
        mbar_init(&wb.bar, 1);
        fence_barrier_init();
    }
    __syncwarp();
    // the first unit of every warp is static (unit = global warp id): no atomic, and nobody can grab two units
    // while a neighbour gets none; its triangles start moving before the descriptor tables are copied
    const uint32_t nwarps_total = gridDim.x * (blockDim.x >> 5);
    uint32_t unit = blockIdx.x + gridDim.x * warp;  // warp w of every CTA before warp w+1 of any: SMs fill evenly
    auto issue_load = [&](uint32_t u) {  // lane 0 only
        const uint32_t t0 = u * a.unit_tris;
        const uint32_t bytes = min(a.unit_tris, a.tri_count - t0) * kTriBytes;
        fence_proxy_async();
        mbar_arrive_expect_tx(&wb.bar, bytes);
        tma_load_1d(wb.tri, tri_bytes + ((size_t)a.tri_first + t0) * kTriBytes, bytes, &wb.bar);
    };
    if (lane == 0 && unit < a.n_units) issue_load(unit);

    // descriptor tables -> shared memory (once per CTA) when they fit
    Tables tabs{a.ranges, a.prims, a.texs, a.nranges};
    {
        const uint32_t br = a.nranges * (uint32_t)sizeof(DRange), bp = a.nprims * (uint32_t)sizeof(DPrim), bt = a.ntex * (uint32_t)sizeof(DTexture);
        if (br + bp + bt <= kTableSmemBytes) {  // uniform across the grid
            unsigned char* base = smem + (size_t)C::kWarps * sizeof(WarpBlock<RK>);
            uint32_t* dst = reinterpret_cast<uint32_t*>(base);  // word-wise: the structs are 16, 56 and 48 bytes
            const uint32_t* s0 = reinterpret_cast<const uint32_t*>(a.ranges);
            const uint32_t* s1 = reinterpret_cast<const uint32_t*>(a.prims);
            const uint32_t* s2 = reinterpret_cast<const uint32_t*>(a.texs);
            const uint32_t n0 = br / 4, n1 = bp / 4, n2 = bt / 4;
            for (uint32_t i = threadIdx.x; i < n0 + n1 + n2; i += blockDim.x)
                dst[i] = i < n0 ? s0[i] : (i < n0 + n1 ? s1[i - n0] : s2[i - n0 - n1]);
            tabs.ranges = reinterpret_cast<const DRange*>(base);
            tabs.prims = reinterpret_cast<const DPrim*>(base + br);
            tabs.texs = reinterpret_cast<const DTexture*>(base + br + bp);
        }
    }
    CtaQueue& cq = *reinterpret_cast<CtaQueue*>(smem + (size_t)C::kWarps * sizeof(WarpBlock<RK>) + kTableSmemBytes);
    if (threadIdx.x == 0) { cq.tail = 0; cq.head = 0; cq.active = blockDim.x >> 5; }
    if (threadIdx.x < kCtaQueueCap) cq.q[threadIdx.x].ready = 0u;
    __syncthreads();  // tables + help queue: the only CTA-wide barrier before the end of the kernel
    // appended launches (m2s_convert_host pipelines a scene in triangle chunks): this launch's records follow those of
    // the earlier chunks; the cap applies to the running index, as the reference's counter does (direct path)
    unsigned long long base_prev = 0;
    for (uint32_t j = 0; j < a.nprev; ++j) base_prev += *reinterpret_cast<const volatile unsigned long long*>(a.prev_totals + j);
    const unsigned long long room = a.cap > base_prev ? a.cap - base_prev : 0ull;
    #ifndef M2S_EXP_NODIRECT
    constexpr bool kDirectOK = (RK == 1);   // PACKED56: the records carry everything the shading needs
#else
    constexpr bool kDirectOK = false;
#endif
    uint32_t phase = 0;
    Stash st;
    st.n_it = 0; st.cur_nb = 0; st.cur_total = 0; st.frags = 0; st.slots = 0; st.seen = 0;
    TR_PHASE(a, kTrEntry);

    while (unit < a.n_units) {
        const uint32_t t0 = unit * a.unit_tris;
        const uint32_t ntri = min(a.unit_tris, a.tri_count - t0);
        uint32_t next = 0xffffffffu;
        // launches with a direct path and fewer than three units per warp: the next unit is claimed only once this unit's
        // work is known (after its shading for a direct unit).  A direct unit shades anything from 0 to 16 groups of 32
        // fragments; claimed up front, every warp would get its two units whatever they weigh, and the kernel would end with
        // the warps that drew heavy ones.  Claimed late, a warp that is still shading leaves the remaining units to the
        // warps that are done.  The late claim costs one exposed atomic round trip per unit: with more units per warp the
        // weights average out and the claim stays up front.  The host decides (ConvertPlan::claim_late).
        const bool claim_late = kDirectOK && a.claim_late != 0;
        if (lane == 0) {
            if (a.n_units > nwarps_total && !claim_late) next = nwarps_total + atomicAdd(SCHED(a, 0), 1u);  // needed only after the set-up
            tma_store_wait_read();  // the previous unit's record store has finished reading wb.rec
        }
        mbar_wait(&wb.bar, phase);
        phase ^= 1;
        __syncwarp();
        TR_PHASE(a, kTrLoadWait);
        TR_ADD(a, kTrUnits, 1);

        // ---- per-triangle stage: one lane per triangle ----
        uint32_t cnt = 0;
        TriSetup ts;
        ts.w = 1; ts.h = 0; ts.incl = 0;
        ts.A[0] = ts.A[1] = ts.A[2] = ts.B[0] = ts.B[1] = ts.B[2] = 0; ts.E0[0] = ts.E0[1] = ts.E0[2] = 0;
        Rec& myrec = wb.rec[lane];
        if ((uint32_t)lane < ntri) cnt = setup_triangle<RK>(wb.tri + lane * 9, a.tri_first + t0 + lane, a, tabs, ts, myrec);
        __syncwarp();
        TR_PHASE(a, kTrSetup);
        next = __shfl_sync(0xffffffffu, next, 0);

        // ---- small triangles: lane-per-triangle lock-step walk of the candidate box -> coverage mask ----
        int e0 = 0, e1 = 0, e2 = 0, a0 = 0, a1 = 0, a2 = 0, r0 = 0, r1 = 0, r2 = 0, w = 1;
        bool small = false;
        if (cnt) {
            w = ts.w;
            const int h = ts.h;
            a0 = ts.A[0]; a1 = ts.A[1]; a2 = ts.A[2];
            const int b0 = ts.B[0], b1 = ts.B[1], b2 = ts.B[2];
            // E at the box origin, with the ownership bias folded in: inside <=> all E' >= 0
            const long long E0 = ts.E0[0] - ((ts.incl & 1u) ? 0 : 1);
            const long long E1 = ts.E0[1] - ((ts.incl & 2u) ? 0 : 1);
            const long long E2 = ts.E0[2] - ((ts.incl & 4u) ? 0 : 1);
            const long long lim = 0x7fffffffll;
            const long long s0 = llabs(E0) + (long long)(w - 1) * abs(a0) + (long long)(h - 1) * abs(b0);
            const long long s1 = llabs(E1) + (long long)(w - 1) * abs(a1) + (long long)(h - 1) * abs(b1);
            const long long s2 = llabs(E2) + (long long)(w - 1) * abs(a2) + (long long)(h - 1) * abs(b2);
            small = cnt <= kSmallCand && h <= 32 && s0 < lim && s1 < lim && s2 < lim;
            if (small) {
                e0 = (int)E0; e1 = (int)E1; e2 = (int)E2;
                r0 = b0 - (w - 1) * a0; r1 = b1 - (w - 1) * a1; r2 = b2 - (w - 1) * a2;  // step to the next row's first pixel
            }
        }
        unsigned long long hits = 0;
        {
            const uint32_t mine = small ? cnt : 0u;
            const uint32_t maxc = __reduce_max_sync(0xffffffffu, mine);
            int col = 0, f0 = e0, f1 = e1, f2 = e2;
            for (uint32_t it = 0; it < maxc; ++it) {
                const bool inside = it < mine && (f0 | f1 | f2) >= 0;
                hits |= (unsigned long long)inside << it;
                if (++col == w) { col = 0; f0 += r0; f1 += r1; f2 += r2; }
                else { f0 += a0; f1 += a1; f2 += a2; }
            }
        }
        const uint32_t nh = (uint32_t)__popcll(hits);
        uint32_t incl_scan = nh;  // inclusive warp scan
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, incl_scan, d);
            if (lane >= d) incl_scan += v;
        }
        const uint32_t total_small = __shfl_sync(0xffffffffu, incl_scan, 31);
        const uint32_t myrows = small ? (uint32_t)ts.h : 0u;  // rows this triangle contributes to the unit item's span table
        uint32_t rows_scan = myrows;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t v = __shfl_up_sync(0xffffffffu, rows_scan, d);
            if (lane >= d) rows_scan += v;
        }
        if ((uint32_t)lane < ntri) {
            myrec.hits = hits;
            myrec.first = (incl_scan - nh) | ((rows_scan - myrows) << 16);
            myrec.box = cnt ? ((unsigned)ts.w | ((unsigned)ts.h << 13) | (ts.incl << 26) | (small ? kBoxSmall : 0u)) : 0u;
        }
        __syncwarp();
        TR_PHASE(a, kTrWalkScan);
        // DIRECT path (REF96 / PACKED56, single GPU): when the unit's small triangles emit at most M2S_DIRECT_MAX fragments
        // this warp shades them itself, straight from the records in its shared-memory slice — no work item, no record
        // round trip through L2, no second kernel on the critical path.  The triangle staging area (dead since the set-up)
        // is the warp's output stage then, so the next unit's triangles start flying in after the shading instead of now.
        const bool direct = kDirectOK && a.direct_ok != 0 && total_small != 0 && total_small <= (uint32_t)M2S_DIRECT_MAX;
        auto claim = [&]() {   // the next unit, claimed once this one's work is known
            if (lane == 0) next = nwarps_total + atomicAdd(SCHED(a, 0), 1u);
            next = __shfl_sync(0xffffffffu, next, 0);
        };
        if (claim_late && !direct) claim();
        if (!direct && lane == 0 && next < a.n_units) issue_load(next);

        // ---- all other triangles: the warp counts one triangle at a time, one lane per pixel row; the tall triangles of
        // a heavy unit are posted to the CTA's help queue instead (see CtaQueue) ----
        const uint32_t gm_all = __ballot_sync(0xffffffffu, cnt != 0 && !small);
        const uint32_t myblocks = (cnt != 0 && !small) ? (uint32_t)(ts.h + 31) / 32u : 0u;
        const uint32_t unit_blocks = __reduce_add_sync(0xffffffffu, myblocks);
        unsigned gm = gm_all;
        if (unit_blocks > kDeferUnitBlocks) {
            unsigned dm = __ballot_sync(0xffffffffu, myblocks >= 2);
            while (dm) {
                const int s = __ffs(dm) - 1;
                dm &= dm - 1;
                int h;
                const RowState rs = row_state(wb.rec[s], h);
                const uint32_t nb = (uint32_t)(h + 31) / 32u, nent = (nb + kDeferBlocks - 1) / kDeferBlocks;
                uint32_t base = 0;
                if (lane == 0) base = atomicAdd_block(&cq.tail, nent);
                base = __shfl_sync(0xffffffffu, base, 0);
                const uint32_t fit = base < kCtaQueueCap ? min(nent, kCtaQueueCap - base) : 0u;  // the first `fit` pieces go to the queue
                if ((uint32_t)lane < fit) {
                    CtaEntry& e = cq.q[base + lane];
                    e.rs = rs; e.h = h; e.unit = unit; e.slot = (uint32_t)s;
                    e.rb0 = lane * kDeferBlocks; e.rb1 = min(nb, (lane + 1) * kDeferBlocks);
                    __threadfence_block();
                    e.ready = 1u;
                }
                if (fit < nent) count_blocks<RK>(a, wb, unit, st, rs, h, (uint32_t)s, (int)(fit * kDeferBlocks), 1 << 20, lane);  // the rest stays here
                gm &= ~(1u << s);
            }
        }
        while (gm) {
            const int s = __ffs(gm) - 1;
            gm &= gm - 1;
            int h;
            const RowState rs = row_state(wb.rec[s], h);  // broadcast reads of the record
            count_blocks<RK>(a, wb, unit, st, rs, h, (uint32_t)s, 0, 1 << 20, lane);
        }
        // ONE atomicAdd per unit (unless the stash filled up on the way) reserves the output range and the queue
        // slots of everything the unit emits
        stash_close_item<RK>(a, wb, unit, st, lane);
        if (!direct) {
            stash_unit_item<RK>(a, wb, unit, st, total_small, ntri, hits, (uint32_t)w, incl_scan - nh, lane);
            stash_flush<RK>(a, wb, unit, st, lane);
        }
        TR_PHASE(a, kTrLarger);
        if constexpr (kDirectOK) {
            if (direct) {
                constexpr int kStride = Cfg<RK>::kStride;   // layout == raster kind for REF96 / PACKED56
                static_assert(32 * kStride <= kUnitTris * kTriBytes, "the output stage lives in the triangle staging area");
                const unsigned long long dfirst = stash_flush<RK>(a, wb, unit, st, lane, total_small);   // the stash area is free after this
                TR_PHASE(a, kTrReserve);
                TR_ADD(a, kTrDirectUnits, 1);
                // every lane lists the covered pixels of its triangle at their place in the unit: slot | column << 5 | row << 11
                unsigned short* list = reinterpret_cast<unsigned short*>(wb.pend);
                {
                    unsigned long long hb = hits;
                    uint32_t k = incl_scan - nh;
                    const uint32_t inv = (65536u + (uint32_t)w - 1u) / (uint32_t)w;  // row = bit / w by a 16.16 reciprocal (exact for bit < 64, w <= 64)
                    while (hb) {
                        const uint32_t b = (uint32_t)__ffsll((long long)hb) - 1u;
                        hb &= hb - 1ull;
                        const uint32_t row = (b * inv) >> 16, col = b - row * (uint32_t)w;
                        list[k++] = (unsigned short)((uint32_t)lane | (col << 5) | (row << 11));
                    }
                }
                __syncwarp();
                TR_PHASE(a, kTrList);
                direct_run<RK>(a, wb, total_small, dfirst, t0, base_prev, room, lane);
                TR_PHASE(a, kTrShade);
                TR_ADD(a, kTrGroups, (total_small + 31) / 32);
                // the stage was written through the generic proxy: every writer fences before the TMA engine writes there again
                fence_proxy_async();
                __syncwarp();
                if (claim_late) claim();
                if (lane == 0 && next < a.n_units) issue_load(next);
            }
        }

        // ---- the unit's records go to global memory for the fragment kernel: one TMA bulk store straight out of
        // this warp's shared-memory slice (every writer fences its generic-proxy writes, then the barrier) ----
        const bool any = __any_sync(0xffffffffu, cnt != 0) && (!direct || gm_all != 0);  // a fully direct unit leaves nothing for the fragment kernel
        if (any) {
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) {
                tma_store_1d(a.tri_frag + (size_t)t0 * sizeof(Rec), wb.rec, ntri * (uint32_t)sizeof(Rec));
                tma_store_commit();
            }
        }
        unit = next;
        TR_PHASE(a, kTrUnitEnd);
    }
    // ---- help: tickets on the CTA's queue until no warp of the CTA can post any more ----
    if (lane == 0) atomicSub_block(&cq.active, 1u);
    for (;;) {
        uint32_t t = 0;
        if (lane == 0) t = atomicAdd_block(&cq.head, 1u);
        t = __shfl_sync(0xffffffffu, t, 0);
        if (t >= kCtaQueueCap) break;  // beyond the capacity nothing is ever posted
        bool have = false;
        if (lane == 0) {
            unsigned ns = 64;   // the waiters must not take issue slots from the warps still working
            for (;;) {
                if (*reinterpret_cast<volatile uint32_t*>(&cq.tail) > t) { have = true; break; }
                if (*reinterpret_cast<volatile uint32_t*>(&cq.active) == 0 && *reinterpret_cast<volatile uint32_t*>(&cq.tail) <= t) break;
                __nanosleep(ns);
                ns = min(ns * 2u, 256u);
            }
            if (have) while (cq.q[t].ready == 0u) __nanosleep(20);
            __threadfence_block();
        }
        if (!__shfl_sync(0xffffffffu, (int)have, 0)) break;
        const CtaEntry& e = cq.q[t];
        const RowState rs = e.rs;
        const int h = e.h;
        const uint32_t eu = e.unit, es = e.slot;
        const int rb0 = (int)e.rb0, rb1 = (int)e.rb1;
        count_blocks<RK>(a, wb, eu, st, rs, h, es, rb0, rb1, lane);
        stash_close_item<RK>(a, wb, eu, st, lane);
        stash_flush<RK>(a, wb, eu, st, lane);
    }
    if (lane == 0) tma_store_wait_all();  // record stores are complete (not just read) before the kernel ends
    // ---- last CTA out publishes the counts and re-arms the scheduler for the next launch ---------
    __syncthreads();
    if (warp == 0) {
        uint32_t last = 0;
        unsigned long long tot = 0;
        if (lane == 0) {
            __threadfence();
            const uint32_t done = atomicAdd(SCHED(a, 4), 1u);
            if (done == gridDim.x - 1) {
                __threadfence();
                last = 1;
                const unsigned long long packed = *reinterpret_cast<volatile unsigned long long*>(a.counter);
                tot = packed & kFragMask;                       // fragments generated
                *a.total_out = tot;
                *a.n_items_out = (uint32_t)(packed >> 40);      // work items queued
                *a.counter = 0ull;
                if (a.host_total) {  // zero-copy count for the host (PCIe posted write, ~1 us)
                    *reinterpret_cast<volatile unsigned long long*>(a.host_total) = tot;
                    __threadfence_system();
                    *reinterpret_cast<volatile unsigned long long*>(a.host_total + 1) = a.host_tag;
                }
                *SCHED(a, 0) = 0; *SCHED(a, 4) = 0;
                __threadfence();
            }
        }
        if (a.world > 1) {  // fused gather: tell every peer how many records this rank will write, one lane per peer
            last = __shfl_sync(0xffffffffu, last, 0);
            tot = __shfl_sync(0xffffffffu, tot, 0);
            if (last && (uint32_t)lane < a.world) {
                const unsigned long long mine = tot < a.cap ? tot : a.cap;
                a.peer_xch[lane][a.rank * 4 + 0] = mine;
                __threadfence_system();
                st_release_sys(a.peer_xch[lane] + a.rank * 4 + 1, a.epoch);
            }
        }
    }
#ifdef M2S_TRACE
    TR_PHASE(a, kTrTail);
    TR_ADD(a, kTrCycles, clock64() - tr_c0_);   // with kTrNanos: the SM clock the cycles convert at
    TR_ADD(a, kTrNanos, gtime() - tr_ns0_);
#endif
}

// A warp's staged records (shared memory) -> one contiguous span of global memory at byte offset `boff` of `dstbase`
// (16-byte aligned).  Strides that are multiples of 16 (REF96, the 48-byte row): 16-byte stores throughout.  Strides
// that are 8 mod 16 (PACKED56, the 248-byte row): a span that starts at an odd record is only 8-byte aligned — the
// caller stages its records 8 bytes into the stage (stage_shift) so that source and destination share the misalignment:
// one 8-byte head, a 16-byte body, one 8-byte tail.  The 76-byte row goes out in 4-byte pieces.
template <int STRIDE>
__device__ __forceinline__ uint32_t stage_shift(unsigned long long record_index) {
    return (STRIDE % 16 == 8) ? (uint32_t)(record_index & 1ull) << 3 : 0u;
}
template <int STRIDE>
__device__ __forceinline__ void copy_span(uint8_t* dstbase, unsigned long long boff, const unsigned char* stage, uint32_t nbytes, int lane) {
    static_assert(STRIDE % 4 == 0, "record strides are multiples of 4");
    if (nbytes == 0) return;
    if (STRIDE % 8 == 0) {
        uint32_t pos = 0;
        if (STRIDE % 16 == 8) {
            stage += (uint32_t)(boff & 8ull);   // == stage_shift of the first record
            if (boff & 8ull) {
                if (lane == 0) *reinterpret_cast<float2*>(dstbase + boff) = *reinterpret_cast<const float2*>(stage);
                pos = 8;
            }
        }
        const uint32_t n16 = (nbytes - pos) / 16;
        float4* dst = reinterpret_cast<float4*>(dstbase + boff + pos);
        const float4* src = reinterpret_cast<const float4*>(stage + pos);
#pragma unroll
        for (int j = 0; j < (32 * STRIDE / 16 + 31) / 32; ++j) {
            const uint32_t c = lane + 32 * j;
            if (c < n16) dst[c] = src[c];
        }
        pos += n16 * 16;
        if (pos < nbytes && lane == 0) *reinterpret_cast<float2*>(dstbase + boff + pos) = *reinterpret_cast<const float2*>(stage + pos);
    } else {
        const uint32_t nw = nbytes / 4;
        uint32_t* dst = reinterpret_cast<uint32_t*>(dstbase + boff);
        const uint32_t* src = reinterpret_cast<const uint32_t*>(stage);
#pragma unroll
        for (int j = 0; j < STRIDE / 4; ++j) {
            const uint32_t c = lane + 32 * j;
            if (c < nw) dst[c] = src[c];
        }
    }
}

// ------------------------------------------------------------------------------------------
// fragment_kernel: one CTA = one work item; one warp step = 32 consecutive fragments = 32 consecutive records
// ------------------------------------------------------------------------------------------
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

__device__ __forceinline__ unsigned char to_byte(float v) {
    v = fminf(fmaxf(v, 0.0f), 1.0f);
    return (unsigned char)roundf(v * 255.0f);
}

// PACKED56 in two halves, so that a warp can have the texel loads of its NEXT 32 fragments in flight while it filters
// and encodes the current ones (direct path of the raster kernel): everything a fragment needs between the halves.
struct Frag1 {
    float Px, Py, Pz, sy;
    float2 w00, w10, w01, w11;   // filter weights: bilinear x 1/255 x level blend, (level 0, level 1)
    uint32_t tx[8];              // RGBA8 texels: level-0 footprint (00, 10, 01, 11), level-1 footprint
    bool has;
};
__device__ __forceinline__ void shade1_fetch(const TriRec<1>& tf, int dxi, int dyi, const uint32_t* __restrict__ texb, Frag1& s) {
    const float2 FX = f2(u2f((uint32_t)dxi)), FY = f2(u2f((uint32_t)dyi));
    const float4* __restrict__ pl = reinterpret_cast<const float4*>(tf.plane);
    const float4 b0 = pl[0], x0 = pl[1], y0 = pl[2], b1 = pl[3];         // (Px, Py, Pz, u) planes; (v, dv/dx, dv/dy, sy)
    const float2 Pzu = ffma2(FY, f2(y0.z, y0.w), ffma2(FX, f2(x0.z, x0.w), f2(b0.z, b0.w)));
    const float2 Pxy = ffma2(FY, f2(y0.x, y0.y), ffma2(FX, f2(x0.x, x0.y), f2(b0.x, b0.y)));
    s.Px = Pxy.x; s.Py = Pxy.y; s.Pz = Pzu.x; s.sy = b1.w;
    const float u = wrap01(Pzu.y), v = wrap01(fmaf(FY.x, b1.z, fmaf(FX.x, b1.y, b1.x)));
    const TexRef ref = tf.tex[0];
    s.has = ref.off0 != 0xffffffffu;
    const float f = tf.frac[0];
    const bool two = s.has && f > 0.0f;
    const Bilin2 bl = bilin_setup2(ref, u, v, f2(1.0f - f, f));
    s.w00 = bl.w00; s.w10 = bl.w10; s.w01 = bl.w01; s.w11 = bl.w11;
    const uint32_t o0 = s.has ? ref.off0 : 0u, o1 = ref.off1;  // uniform base + 32-bit texel index
    s.tx[0] = s.has ? __ldg(texb + (o0 + bl.i00[0])) : 0u; s.tx[1] = s.has ? __ldg(texb + (o0 + bl.i10[0])) : 0u;
    s.tx[2] = s.has ? __ldg(texb + (o0 + bl.i01[0])) : 0u; s.tx[3] = s.has ? __ldg(texb + (o0 + bl.i11[0])) : 0u;
    s.tx[4] = two ? __ldg(texb + (o1 + bl.i00[1])) : 0u; s.tx[5] = two ? __ldg(texb + (o1 + bl.i10[1])) : 0u;
    s.tx[6] = two ? __ldg(texb + (o1 + bl.i01[1])) : 0u; s.tx[7] = two ? __ldg(texb + (o1 + bl.i11[1])) : 0u;
}
template <int CH>
__device__ __forceinline__ float filt2s(const Frag1& s, uint32_t k4b) {
    float2 acc = fmul2(s.w00, tex_ch2<CH>(s.tx[0], s.tx[4], k4b));
    acc = ffma2(s.w10, tex_ch2<CH>(s.tx[1], s.tx[5], k4b), acc);
    acc = ffma2(s.w01, tex_ch2<CH>(s.tx[2], s.tx[6], k4b), acc);
    acc = ffma2(s.w11, tex_ch2<CH>(s.tx[3], s.tx[7], k4b), acc);
    return acc.x + acc.y;
}
__device__ __forceinline__ void shade1_finish(const ConvertArgs& a, const TriRec<1>& tf, const Frag1& s, unsigned char* __restrict__ srec_bytes) {
    // converterFS.glsl:55-62,99; parsers.cpp:484-499: SH0, opacity logit, log scale (per triangle)
    const uint32_t k4b = opaque_4b();
    float cr = 1.f, cg = 1.f, cb = 1.f, ca = 1.f;
    if (s.has) { cr = filt2s<0>(s, k4b); cg = filt2s<1>(s, k4b); cb = filt2s<2>(s, k4b); ca = filt2s<3>(s, k4b); }
    const float4 q = *reinterpret_cast<const float4*>(tf.quat), fc = *reinterpret_cast<const float4*>(tf.factor);
    cr *= fc.x; cg *= fc.y; cb *= fc.z; ca *= fc.w;
    float2* s2 = reinterpret_cast<float2*>(srec_bytes);
    s2[0] = make_float2(s.Px, s.Py);
    s2[1] = make_float2(s.Pz, q.x);
    s2[2] = make_float2(q.y, q.z);
    s2[3] = make_float2(q.w, tf.sx);
    s2[4] = make_float2(s.sy, a.log_sz);
    s2[5] = make_float2(sh0_encode(cr), sh0_encode(cg));
    s2[6] = make_float2(sh0_encode(cb), opacity_logit(ca));
}

// One fragment: pixel (dx, dy) relative to the box origin of the triangle whose record is `tf`; v: its 9 float4 of vertex
// data (three-map layouts; unused by PACKED56).
template <int LAYOUT>
__device__ __forceinline__ void shade(const ConvertArgs& a, const TriRec<RCfg<Cfg<LAYOUT>::kRK>::kMaps>& tf, const float4* __restrict__ v,
                                      int dxi, int dyi, const uint32_t* __restrict__ texb, unsigned char* __restrict__ srec_bytes) {
    constexpr int kMaps = RCfg<Cfg<LAYOUT>::kRK>::kMaps;
    if constexpr (LAYOUT == 1) {   // PACKED56: planes in the record, no vertices
        Frag1 s;
        shade1_fetch(tf, dxi, dyi, texb, s);
        shade1_finish(a, tf, s, srec_bytes);
    } else {
    const uint32_t k4b = opaque_4b();
    const float ia = tf.inv_area;
    const float l0 = __ll2float_rn(tf.E0[0] + (long long)tf.A[0] * dxi + (long long)tf.B[0] * dyi) * ia;
    const float l1 = __ll2float_rn(tf.E0[1] + (long long)tf.A[1] * dxi + (long long)tf.B[1] * dyi) * ia;
    const float l2 = __ll2float_rn(tf.E0[2] + (long long)tf.A[2] * dxi + (long long)tf.B[2] * dyi) * ia;
    const float2 L0 = f2(l0), L1 = f2(l1), L2 = f2(l2);
    // vertices: 3 x {pos3 nrm3 tan4 uv2} = 9 float4 in shared memory; attribute pairs are interpolated as float2 pairs
    const float4 a2 = v[2], b2 = v[5], c2 = v[8];
    auto lerp3 = [&](float2 A, float2 B, float2 C) { return ffma2(L2, C, ffma2(L1, B, fmul2(L0, A))); };
    // uv first: the texel addresses depend on nothing else
    const float2 uv = lerp3(f2(a2.z, a2.w), f2(b2.z, b2.w), f2(c2.z, c2.w));
    const float u = wrap01(uv.x), vv = wrap01(uv.y);
    const unsigned meta = tf.meta;

    // ---- issue every texel load of every bound map back to back ----
    uint32_t tx[kMaps][8];
    Bilin2 bl[kMaps];
    bool has[kMaps];
#pragma unroll
    for (int m = 0; m < kMaps; ++m) {
        const TexRef ref = tf.tex[m];
        has[m] = ref.off0 != 0xffffffffu;
        const float f = tf.frac[m];
        const bool two = has[m] && f > 0.0f;
        if (m == 0 || !((meta >> m) & 1u)) bl[m] = bilin_setup2(ref, u, vv, f2(1.0f - f, f));
        else bl[m] = bl[0];  // same level sizes and blend as map 0: same footprint and weights
        const uint32_t o0 = has[m] ? ref.off0 : 0u, o1 = ref.off1;  // uniform base + 32-bit texel index
        tx[m][0] = has[m] ? __ldg(texb + (o0 + bl[m].i00[0])) : 0u; tx[m][1] = has[m] ? __ldg(texb + (o0 + bl[m].i10[0])) : 0u;
        tx[m][2] = has[m] ? __ldg(texb + (o0 + bl[m].i01[0])) : 0u; tx[m][3] = has[m] ? __ldg(texb + (o0 + bl[m].i11[0])) : 0u;
        tx[m][4] = two ? __ldg(texb + (o1 + bl[m].i00[1])) : 0u; tx[m][5] = two ? __ldg(texb + (o1 + bl[m].i10[1])) : 0u;
        tx[m][6] = two ? __ldg(texb + (o1 + bl[m].i01[1])) : 0u; tx[m][7] = two ? __ldg(texb + (o1 + bl[m].i11[1])) : 0u;
    }
    // ---- interpolate the remaining varyings while the loads are in flight ----
    const float4 a0 = v[0], b0 = v[3], c0 = v[6];
    const float2 Pxy = lerp3(f2(a0.x, a0.y), f2(b0.x, b0.y), f2(c0.x, c0.y));
    const float2 PzNx = lerp3(f2(a0.z, a0.w), f2(b0.z, b0.w), f2(c0.z, c0.w));
    const float Px = Pxy.x, Py = Pxy.y, Pz = PzNx.x;

    // colour (converterFS.glsl:55-62,99): the level blend is part of the weights, a single-level lookup has weight 0
    // (and no loads) on the second level
    float cr = 1.f, cg = 1.f, cb = 1.f, ca = 1.f;
    if (has[0]) {
        cr = filt2<0>(bl[0], tx[0], k4b); cg = filt2<1>(bl[0], tx[0], k4b); cb = filt2<2>(bl[0], tx[0], k4b); ca = filt2<3>(bl[0], tx[0], k4b);
    }
    cr *= tf.factor[0]; cg *= tf.factor[1]; cb *= tf.factor[2]; ca *= tf.factor[3];

    // ---- every other layout carries the shading normal; PBR values where the layout has them ----
    constexpr int MN = kMaps > 1 ? 1 : 0, MM = kMaps > 2 ? 2 : 0;
    const float Nx = PzNx.y;
    const float4 a1 = v[1], b1 = v[4], c1 = v[7];
    const float2 Nyz = lerp3(f2(a1.x, a1.y), f2(b1.x, b1.y), f2(c1.x, c1.y));
    const float Ny = Nyz.x, Nz = Nyz.y;
    float nx = Nx, ny = Ny, nz = Nz;
    if (has[MN]) {  // :64-77 TBN
        const float mx = filt2<0>(bl[MN], tx[MN], k4b), my = filt2<1>(bl[MN], tx[MN], k4b), mz = filt2<2>(bl[MN], tx[MN], k4b);
        const float2 Txy = lerp3(f2(a1.z, a1.w), f2(b1.z, b1.w), f2(c1.z, c1.w));
        const float2 Tzw = lerp3(f2(a2.x, a2.y), f2(b2.x, b2.y), f2(c2.x, c2.y));
        const float Tx = Txy.x, Ty = Txy.y, Tz = Tzw.x, Tw = Tzw.y;
        float rx = mx * 2.0f - 1.0f, ry = my * 2.0f - 1.0f, rz = mz * 2.0f - 1.0f;
        float inv = rsqrtf(rx * rx + ry * ry + rz * rz);
        rx *= inv; ry *= inv; rz *= inv;
        float bx = Ny * Tz - Ty * Nz, by = Nz * Tx - Tz * Nx, bz = Nx * Ty - Tx * Ny;  // cross(N,T)
        inv = Tw * rsqrtf(bx * bx + by * by + bz * bz);
        bx *= inv; by *= inv; bz *= inv;
        inv = rsqrtf(Nx * Nx + Ny * Ny + Nz * Nz);
        const float ox = Tx * rx + bx * ry + Nx * inv * rz, oy = Ty * rx + by * ry + Ny * inv * rz,
                    oz = Tz * rx + bz * ry + Nz * inv * rz;
        inv = rsqrtf(ox * ox + oy * oy + oz * oz);
        nx = ox * inv; ny = oy * inv; nz = oz * inv;
    }
    float metal = 0.1f, rough = 0.5f;  // :83-95 (.bg)
    if (LAYOUT != 2 && has[MM]) {      // the standard .ply row carries no PBR values
        rough = filt2<1>(bl[MM], tx[MM], k4b);
        metal = filt2<2>(bl[MM], tx[MM], k4b);
    }
    if (LAYOUT == 0) {
        float4* s4 = reinterpret_cast<float4*>(srec_bytes);
        s4[0] = make_float4(Px, Py, Pz, 1.0f);
        s4[1] = make_float4(cr, cg, cb, ca);
        s4[2] = make_float4(tf.sx, tf.sy, 1e-7f, 0.0f);
        s4[3] = make_float4(nx, ny, nz, 0.0f);
        s4[4] = make_float4(tf.quat[0], tf.quat[1], tf.quat[2], tf.quat[3]);
        s4[5] = make_float4(metal, rough, 0.0f, 1.0f);
    } else if (LAYOUT == 2) {  // parsers.cpp:431-514: xyz n f_dc f_rest(45 x 0) opacity scale rot — 62 floats, 8-byte aligned rows
        float2* s2 = reinterpret_cast<float2*>(srec_bytes);
        s2[0] = make_float2(Px, Py); s2[1] = make_float2(Pz, nx); s2[2] = make_float2(ny, nz);
        s2[3] = make_float2(sh0_encode(cr), sh0_encode(cg));
        s2[4] = make_float2(sh0_encode(cb), 0.0f);
#pragma unroll
        for (int k = 5; k < 27; ++k) s2[k] = make_float2(0.0f, 0.0f);
        s2[27] = make_float2(opacity_logit(ca), tf.sx);
        s2[28] = make_float2(tf.sy, a.log_sz);
        s2[29] = make_float2(tf.quat[0], tf.quat[1]);
        s2[30] = make_float2(tf.quat[2], tf.quat[3]);
    } else if (LAYOUT == 3) {  // parsers.cpp:232-316: 19 floats, 4-byte aligned rows
        float* f = reinterpret_cast<float*>(srec_bytes);
        f[0] = Px; f[1] = Py; f[2] = Pz; f[3] = nx; f[4] = ny; f[5] = nz;
        f[6] = sh0_encode(cr); f[7] = sh0_encode(cg); f[8] = sh0_encode(cb);
        f[9] = metal; f[10] = rough; f[11] = opacity_logit(ca);
        f[12] = tf.sx; f[13] = tf.sy; f[14] = a.log_sz;
        f[15] = tf.quat[0]; f[16] = tf.quat[1]; f[17] = tf.quat[2]; f[18] = tf.quat[3];
    } else {                   // parsers.cpp:339-428: 48-byte rows
        float* f = reinterpret_cast<float*>(srec_bytes);
        unsigned char* p = srec_bytes;
        f[0] = Px; f[1] = Py; f[2] = Pz;
        *reinterpret_cast<uchar4*>(p + 12) = make_uchar4(to_byte(cr), to_byte(cg), to_byte(cb), to_byte(ca));
        f[4] = tf.quat[0]; f[5] = tf.quat[1]; f[6] = tf.quat[2]; f[7] = tf.quat[3];
        f[8] = tf.sx; f[9] = tf.sy; f[10] = fminf(tf.sx, tf.sy);  // log(min(sx,sy) * mult): log is monotonic
        // octahedral normal (parsers.cpp:318-337)
        // (no contraction: the bytes equal the writer's on the same normal, ply_rows_kernel)
        const float s = __fadd_rn(__fadd_rn(__fadd_rn(fabsf(nx), fabsf(ny)), fabsf(nz)), 1e-8f);
        const float ox = __fdiv_rn(nx, s), oy = __fdiv_rn(ny, s), oz = __fdiv_rn(nz, s);
        float rx, ry;
        if (oz >= 0.0f) { rx = ox; ry = oy; }
        else {
            const float m = (ox >= 0.0f && oy >= 0.0f) ? 1.0f : -1.0f;
            rx = __fmul_rn(__fsub_rn(1.0f, fabsf(oy)), m); ry = __fmul_rn(__fsub_rn(1.0f, fabsf(ox)), m);
        }
        const float qx = fminf(fmaxf(roundf(__fmul_rn(__fadd_rn(__fmul_rn(rx, 0.5f), 0.5f), 255.0f)), 0.0f), 255.0f);
        const float qy = fminf(fmaxf(roundf(__fmul_rn(__fadd_rn(__fmul_rn(ry, 0.5f), 0.5f), 255.0f)), 0.0f), 255.0f);
        *reinterpret_cast<uchar4*>(p + 44) = make_uchar4((unsigned char)qx, (unsigned char)qy, to_byte(rough), to_byte(metal));
    }
    }   // three-map layouts
}

// The direct path's worker: the `total` listed fragments of this warp's unit, 32 at a time.  Out of line: its registers
// are not the raster loop's.
template <int RK>
__device__ __noinline__ void direct_run(const ConvertArgs& a, WarpBlock<RK>& wb, uint32_t total, unsigned long long dfirst, uint32_t t0,
                                        unsigned long long base_prev, unsigned long long room, int lane) {
    constexpr int kStride = Cfg<RK>::kStride;   // layout == raster kind for REF96 / PACKED56
    static_assert(32 * kStride <= kUnitTris * kTriBytes, "the output stage lives in the triangle staging area");
    unsigned char* stage = reinterpret_cast<unsigned char*>(wb.tri);   // dead since the set-up of the unit
    const unsigned short* list = reinterpret_cast<const unsigned short*>(wb.pend);
    for (uint32_t g0 = 0; g0 < total; g0 += 32) {
        const uint32_t nfr = min(32u, total - g0);
        const uint32_t e = list[g0 + min((uint32_t)lane, nfr - 1u)];  // idle lanes shadow the last fragment
        const uint32_t slot = e & 31u;
        const int dxi = (int)((e >> 5) & 63u), dyi = (int)(e >> 11);
        const unsigned long long idx0 = dfirst + g0;
        shade<RK>(a, wb.rec[slot], nullptr, dxi, dyi, a.tex_base, stage + stage_shift<kStride>(base_prev + idx0) + lane * kStride);
        __syncwarp();
        uint32_t nval = 0;
        if (idx0 < room) nval = (uint32_t)min((unsigned long long)nfr, room - idx0);
        copy_span<kStride>(a.out, (base_prev + idx0) * (unsigned long long)kStride, stage, nval * kStride, lane);
        if (a.keys != nullptr && (uint32_t)lane < nval) {
            const unsigned meta = wb.rec[slot].meta;
            const unsigned long long tg = a.tri_first + t0 + slot;
            a.keys[base_prev + idx0 + lane] = (tg << 24) | ((unsigned long long)(((meta >> 16) & 0xfffu) + (unsigned)dyi) << 12) |
                                              (unsigned long long)(((meta >> 4) & 0xfffu) + (unsigned)dxi);
        }
        __syncwarp();
    }
}

// A micro item (kItMicro): <= 32 fragments listed in the item itself, shaded by one warp with direct loads.  Out of line:
// the second copy of the shading code must not add to the register pressure of the main loop.
template <int LAYOUT>
__device__ __noinline__ void micro_item(const ConvertArgs& a, uint32_t it, uint4 h0, uint32_t nfr, unsigned long long base, unsigned long long room,
                                        unsigned long long goff, const uint32_t* __restrict__ texb, unsigned char* stage, int lane) {
    using Rec = typename FragSmem<LAYOUT>::Rec;
    constexpr int kStride = Cfg<LAYOUT>::kStride;
    const unsigned long long first = (unsigned long long)h0.x | ((unsigned long long)h0.y << 32);
    const uint32_t t0 = h0.z * a.unit_tris;
    const uint32_t w32 = __ldg(reinterpret_cast<const uint32_t*>((a.items + it)->blocks) + min((uint32_t)lane, nfr - 1u));  // idle lanes shadow the last fragment
    const uint32_t slot = w32 & 31u;
    const Rec* tfp = reinterpret_cast<const Rec*>(a.tri_frag) + (size_t)t0 + slot;
    const unsigned long long mrec = a.world <= 1 ? base + first : goff + first;   // first record of the span in its destination
    shade<LAYOUT>(a, *tfp, a.tris + ((size_t)a.tri_first + t0 + slot) * 9, (int)((w32 >> 5) & 63u), (int)((w32 >> 11) & 63u), texb,
                  stage + stage_shift<kStride>(mrec) + lane * kStride);  
    __syncwarp();
    uint32_t nval = 0;
    if (first < room) nval = (uint32_t)min((unsigned long long)nfr, room - first);
    if (a.world <= 1) {
        copy_span<kStride>(a.out, (base + first) * (unsigned long long)kStride, stage, nval * kStride, lane);
    } else {
        const unsigned long long gbase = goff + first;
        uint32_t gval = 0;
        if (gbase < a.gcap) gval = (uint32_t)min((unsigned long long)nval, a.gcap - gbase);
        uint32_t p = (a.rank + 1u + it) % a.world;
        for (uint32_t i = 0; i < a.world; ++i) {
            copy_span<kStride>(a.peer_out[p], gbase * (unsigned long long)kStride, stage, gval * kStride, lane);
            p = p + 1 == a.world ? 0 : p + 1;
        }
    }
    if (a.keys != nullptr && (uint32_t)lane < nval) {
        const unsigned meta = tfp->meta;
        const unsigned long long tg = a.tri_first + t0 + slot;
        a.keys[base + first + lane] = (tg << 24) | ((unsigned long long)(((meta >> 16) & 0xfffu) + ((w32 >> 11) & 63u)) << 12) |
                                      (unsigned long long)(((meta >> 4) & 0xfffu) + ((w32 >> 5) & 63u));
    }
    __syncwarp();
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
    // launched with programmatic stream serialisation: the CTAs of this grid are placed while the raster
    // kernel drains; everything it wrote is visible after this wait
    asm volatile("griddepcontrol.wait;" ::: "memory");
    // appended launches (m2s_convert_host pipelines a scene in triangle chunks): this launch's records follow
    // those of the earlier chunks; the cap applies to the running index, as the reference's counter does
    unsigned long long base = 0;
    for (uint32_t j = 0; j < a.nprev; ++j) base += *reinterpret_cast<const volatile unsigned long long*>(a.prev_totals + j);
    const unsigned long long room = a.cap > base ? a.cap - base : 0ull;
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
    const bool want_keys = a.keys != nullptr;
    // ---- the item pipeline: header + block list of item i+1 are loaded while item i is processed, and (2 buffers) its
    // records and vertices are already in flight (TMA) into the other staged-unit buffer ----
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
    auto live = [&](const Hdr& h) {  // uniform over the CTA: does the item emit anything?
        const unsigned long long first = (unsigned long long)h.h0.x | ((unsigned long long)h.h0.y << 32);
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
    // the first header is loaded together with the item count (one global round trip instead of two before the first
    // TMA): whatever an unused queue slot holds is discarded by the loop condition
    Hdr cur = load_hdr(blockIdx.x, a.queue_cap);
    const uint32_t nitems = min(*reinterpret_cast<const volatile uint32_t*>(a.n_items_out), a.queue_cap);
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
        const unsigned long long first = (unsigned long long)cur.h0.x | ((unsigned long long)cur.h0.y << 32);
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
                const Rec& r = recs[slot];
                const unsigned box = r.box;
                uint32_t n = 0;
                int xl = 0;
                if ((uint32_t)lane < nrows) {
                    RowState rs;
#pragma unroll
                    for (int k = 0; k < 3; ++k) {
                        rs.E[k] = r.E0[k] - (((box >> (26 + k)) & 1u) ? 0 : 1);
                        rs.A[k] = r.A[k]; rs.B[k] = r.B[k];
                    }
                    rs.w = (int)(box & 0x1fffu);
                    n = span_row(rs, (int)(row_begin + lane), xl);
                }
                uint32_t incl = n;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const uint32_t t = __shfl_up_sync(0xffffffffu, incl, d);
                    if (lane >= d) incl += t;
                }
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
            // ---- the warp's records are one contiguous span: straight vector copy -----------------------
            uint32_t nval = 0;
            if (idx0 < room) nval = (uint32_t)min((unsigned long long)nfr, room - idx0);
            if (a.world <= 1) {
                copy_span<kStride>(a.out, (base + idx0) * (unsigned long long)kStride, stage, nval * kStride, lane);
            } else {
                // fused gather: the same span goes to the final buffer of EVERY rank (peer stores over NVLink)
                const unsigned long long gbase = goff + idx0;
                uint32_t gval = 0;
                if (gbase < a.gcap) gval = (uint32_t)min((unsigned long long)nval, a.gcap - gbase);
                // destinations are visited in a rotated order (by rank and by span) so that at any moment the
                // grid's stores are spread over all peers' ingress ports instead of converging on peer 0
                uint32_t p = (a.rank + 1u + it + g) % a.world;
                for (uint32_t i = 0; i < a.world; ++i) {
                    copy_span<kStride>(a.peer_out[p], gbase * (unsigned long long)kStride, stage, gval * kStride, lane);
                    p = p + 1 == a.world ? 0 : p + 1;
                }
            }
            if (want_keys && (uint32_t)lane < nval) {  // fragment identity: triangle << 24 | y << 12 | x
                const unsigned meta = tf.meta;
                const unsigned long long tg = a.tri_first + t0 + slot;
                a.keys[base + idx0 + lane] = (tg << 24) | ((unsigned long long)(((meta >> 16) & 0xfffu) + (unsigned)dyi) << 12) |
                                             (unsigned long long)(((meta >> 4) & 0xfffu) + (unsigned)dxi);
            }
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
}

// waits until every rank's records of this epoch have landed in THIS rank's final buffer, publishes the
// total; one thread — the data path never returns to the host
__global__ void gather_wait_kernel(const unsigned long long* xch, uint32_t world, unsigned long long epoch,
                                   unsigned long long gcap, unsigned long long* total_global, uint32_t* status) {
    unsigned long long tot = 0;
    for (uint32_t r = 0; r < world; ++r) {
        wait_epoch(xch + r * 4 + 2, epoch, status, 2u);
        tot += *reinterpret_cast<const volatile unsigned long long*>(xch + r * 4);
    }
    if (total_global) *total_global = tot;
    (void)gcap;
}

// ------------------------------------------------------------------------------------------
// mip chain: 2x2 box, round half up (matches oracle orc_mip_down; GL_TEXTURE_MAX_LEVEL 4, glUtils.cpp:313)
// ------------------------------------------------------------------------------------------
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

// ------------------------------------------------------------------------------------------
// v-range of a triangle range per texture (host pipeline: which texture rows must be uploaded before these triangles
// can be shaded).  minmax: [ntex] sortable-int minima | [ntex] maxima | 1 flag (non-finite or absurd v seen).
// ------------------------------------------------------------------------------------------
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

// ------------------------------------------------------------------------------------------
// .ply body rows from REF96 records (parsers.cpp:232-316,339-428,431-514)
// ------------------------------------------------------------------------------------------
__global__ void ply_rows_kernel(const float4* __restrict__ rec, unsigned long long count,
                                const unsigned long long* __restrict__ d_count, uint32_t format, float mult,
                                unsigned char* __restrict__ rows) {
    const unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (d_count) count = min(count, *d_count);  // device-side count (enqueue-only path)
    if (i >= count) return;
    const float4 pos = rec[i * 6 + 0], col = rec[i * 6 + 1], sc = rec[i * 6 + 2], nrm = rec[i * 6 + 3], rot = rec[i * 6 + 4],
                 pbr = rec[i * 6 + 5];
    const float sh0 = sh0_encode(col.x), sh1 = sh0_encode(col.y), sh2 = sh0_encode(col.z);
    const float op = opacity_logit(col.w);
    const float lx = log_scale(sc.x, mult), ly = log_scale(sc.y, mult), lz = log_scale(sc.z, mult);
    if (format == 1) {
        float* f = reinterpret_cast<float*>(rows + i * 76ull);
        f[0] = pos.x; f[1] = pos.y; f[2] = pos.z; f[3] = nrm.x; f[4] = nrm.y; f[5] = nrm.z;
        f[6] = sh0; f[7] = sh1; f[8] = sh2; f[9] = pbr.x; f[10] = pbr.y; f[11] = op;
        f[12] = lx; f[13] = ly; f[14] = lz; f[15] = rot.x; f[16] = rot.y; f[17] = rot.z; f[18] = rot.w;
    } else if (format == 2) {
        unsigned char* p = rows + i * 48ull;
        float* f = reinterpret_cast<float*>(p);
        f[0] = pos.x; f[1] = pos.y; f[2] = pos.z;
        p[12] = to_byte(col.x); p[13] = to_byte(col.y); p[14] = to_byte(col.z); p[15] = to_byte(col.w);
        f[4] = rot.x; f[5] = rot.y; f[6] = rot.z; f[7] = rot.w;
        const float mn = (sc.y < sc.x) ? sc.y : sc.x;
        f[8] = lx; f[9] = ly; f[10] = log_scale(mn, mult);
        // octahedral normal (parsers.cpp:318-337)
        const float s = __fadd_rn(__fadd_rn(__fadd_rn(fabsf(nrm.x), fabsf(nrm.y)), fabsf(nrm.z)), 1e-8f);
        const float nx = __fdiv_rn(nrm.x, s), ny = __fdiv_rn(nrm.y, s), nz = __fdiv_rn(nrm.z, s);
        float rx, ry;
        if (nz >= 0.0f) { rx = nx; ry = ny; }
        else {
            const float m = (nx >= 0.0f && ny >= 0.0f) ? 1.0f : -1.0f;
            rx = __fmul_rn(__fsub_rn(1.0f, fabsf(ny)), m); ry = __fmul_rn(__fsub_rn(1.0f, fabsf(nx)), m);
        }
        const float ox = __fadd_rn(__fmul_rn(rx, 0.5f), 0.5f), oy = __fadd_rn(__fmul_rn(ry, 0.5f), 0.5f);
        p[44] = (unsigned char)fminf(fmaxf(roundf(__fmul_rn(ox, 255.0f)), 0.0f), 255.0f);
        p[45] = (unsigned char)fminf(fmaxf(roundf(__fmul_rn(oy, 255.0f)), 0.0f), 255.0f);
        p[46] = to_byte(pbr.y); p[47] = to_byte(pbr.x);
    } else {
        float* f = reinterpret_cast<float*>(rows + i * 248ull);
        f[0] = pos.x; f[1] = pos.y; f[2] = pos.z; f[3] = nrm.x; f[4] = nrm.y; f[5] = nrm.z;
        f[6] = sh0; f[7] = sh1; f[8] = sh2;
        for (int k = 9; k < 54; ++k) f[k] = 0.0f;
        f[54] = op; f[55] = lx; f[56] = ly; f[57] = lz; f[58] = rot.x; f[59] = rot.y; f[60] = rot.z; f[61] = rot.w;
    }
}

// ------------------------------------------------------------------------------------------
// launch wrappers used by the host code (m2s_scene.cu, m2s_convert.cu), declared in m2s_device.cuh
// ------------------------------------------------------------------------------------------
static int raster_kind(int layout) { return layout == 0 ? 0 : (layout == 1 ? 1 : 2); }
static_assert(sizeof(WarpBlock<0>) * RCfg<0>::kWarps + kTableSmemBytes + sizeof(CtaQueue) <= 232448 &&
              sizeof(WarpBlock<1>) * RCfg<1>::kWarps + kTableSmemBytes + sizeof(CtaQueue) <= 232448 &&
              sizeof(WarpBlock<2>) * RCfg<2>::kWarps + kTableSmemBytes + sizeof(CtaQueue) <= 232448, "raster kernel: 227 KB of shared memory per CTA");
size_t raster_smem_bytes(int layout) {
    const int rk = raster_kind(layout);
    const size_t wb = rk == 0 ? sizeof(WarpBlock<0>) * RCfg<0>::kWarps : (rk == 1 ? sizeof(WarpBlock<1>) * RCfg<1>::kWarps : sizeof(WarpBlock<2>) * RCfg<2>::kWarps);
    return wb + kTableSmemBytes + sizeof(CtaQueue);
}
size_t fragment_smem_bytes(int layout) {
    switch (layout) {
        case 0: return FragSmem<0>::kBytes;
        case 1: return FragSmem<1>::kBytes;
        case 2: return FragSmem<2>::kBytes;
        case 3: return FragSmem<3>::kBytes;
        default: return FragSmem<4>::kBytes;
    }
}
int convert_warps_per_cta(int layout) { const int rk = raster_kind(layout); return rk == 0 ? RCfg<0>::kWarps : (rk == 1 ? RCfg<1>::kWarps : RCfg<2>::kWarps); }
size_t tri_frag_bytes(int layout) { return raster_kind(layout) == 1 ? sizeof(TriRec<1>) : sizeof(TriRec<3>); }

template <int RK>
static cudaError_t configure_raster(size_t smem, int* blocks) {
    cudaError_t e = cudaFuncSetAttribute(raster_kernel<RK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    return cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks, raster_kernel<RK>, RCfg<RK>::kWarps * 32, smem);
}
template <int L>
static cudaError_t configure_fragment(size_t smem, int* blocks) {
    cudaError_t e = cudaFuncSetAttribute(fragment_kernel<L>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    return cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks, fragment_kernel<L>, kFragThreads, smem);
}

cudaError_t convert_configure(int layout, int* raster_blocks_per_sm, int* fragment_blocks_per_sm) {
    const size_t smem = raster_smem_bytes(layout), fsmem = fragment_smem_bytes(layout);
    cudaError_t e;
    switch (raster_kind(layout)) {
        case 0: e = configure_raster<0>(smem, raster_blocks_per_sm); break;
        case 1: e = configure_raster<1>(smem, raster_blocks_per_sm); break;
        default: e = configure_raster<2>(smem, raster_blocks_per_sm); break;
    }
    if (e != cudaSuccess) return e;
    switch (layout) {
        case 0: return configure_fragment<0>(fsmem, fragment_blocks_per_sm);
        case 1: return configure_fragment<1>(fsmem, fragment_blocks_per_sm);
        case 2: return configure_fragment<2>(fsmem, fragment_blocks_per_sm);
        case 3: return configure_fragment<3>(fsmem, fragment_blocks_per_sm);
        default: return configure_fragment<4>(fsmem, fragment_blocks_per_sm);
    }
}

// mid != nullptr: record it between the two kernels (measurement of the per-kernel shares; disables the programmatic
// dependent launch, so the kernels do not overlap)
cudaError_t convert_launch(int layout, const ConvertArgs& args, int raster_grid, int fragment_grid, cudaStream_t stream, cudaEvent_t mid) {
    const size_t smem = raster_smem_bytes(layout), fsmem = fragment_smem_bytes(layout);
    switch (raster_kind(layout)) {
        case 0: raster_kernel<0><<<raster_grid, RCfg<0>::kWarps * 32, smem, stream>>>(args); break;
        case 1: raster_kernel<1><<<raster_grid, RCfg<1>::kWarps * 32, smem, stream>>>(args); break;
        default: raster_kernel<2><<<raster_grid, RCfg<2>::kWarps * 32, smem, stream>>>(args); break;
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    if (mid) { e = cudaEventRecord(mid, stream); if (e != cudaSuccess) return e; }
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)fragment_grid);
    cfg.blockDim = dim3(kFragThreads);
    cfg.dynamicSmemBytes = fsmem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;  // PDL: overlap this launch with the raster kernel's tail
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
#ifndef M2S_NO_PDL
    cfg.numAttrs = mid ? 0 : 1;
#else
    cfg.numAttrs = 0;
#endif
    switch (layout) {
        case 0: return cudaLaunchKernelEx(&cfg, fragment_kernel<0>, args);
        case 1: return cudaLaunchKernelEx(&cfg, fragment_kernel<1>, args);
        case 2: return cudaLaunchKernelEx(&cfg, fragment_kernel<2>, args);
        case 3: return cudaLaunchKernelEx(&cfg, fragment_kernel<3>, args);
        default: return cudaLaunchKernelEx(&cfg, fragment_kernel<4>, args);
    }
}

cudaError_t gather_wait_launch(const unsigned long long* xch, uint32_t world, unsigned long long epoch, unsigned long long gcap,
                               unsigned long long* total_global, uint32_t* status, cudaStream_t stream) {
    gather_wait_kernel<<<1, 1, 0, stream>>>(xch, world, epoch, gcap, total_global, status);
    return cudaGetLastError();
}

// levels 1.. of the 16-row groups [g0, g1) of one texture (level 0 must be resident), one launch
cudaError_t mip_groups_launch(uint32_t* arena, const DTexture& t, uint32_t g0, uint32_t g1, cudaStream_t stream) {
    if (t.nlevels <= 1 || g1 <= g0) return cudaSuccess;
    dim3 grd((t.w[0] + 63) / 64, g1 - g0);
    mip_groups_kernel<<<grd, 256, 0, stream>>>(arena, t, g0);
    return cudaGetLastError();
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
cudaError_t vrange_publish_launch(int* minmax, uint32_t ntex, int* host, unsigned long long* host_tag, unsigned long long tag, cudaStream_t stream) {
    vrange_publish_kernel<<<1, 128, 0, stream>>>(minmax, ntex, host, host_tag, tag);
    return cudaGetLastError();
}

cudaError_t vrange_launch(const float4* tris, uint32_t first, uint32_t count, const DRange* ranges, uint32_t nranges, const DPrim* prims,
                          uint32_t ntex, int* minmax, cudaStream_t stream) {
    if (!count || !ntex) return cudaSuccess;
    vrange_kernel<<<(count + 255) / 256, 256, 0, stream>>>(tris, first, count, ranges, nranges, prims, ntex, minmax);
    return cudaGetLastError();
}

cudaError_t ply_rows_launch(const void* ref96, unsigned long long count, const unsigned long long* d_count,
                            uint32_t format, float mult, void* rows, cudaStream_t stream) {
    if (count == 0) return cudaSuccess;
    const unsigned blocks = (unsigned)((count + 255) / 256);
    ply_rows_kernel<<<blocks, 256, 0, stream>>>(reinterpret_cast<const float4*>(ref96), count, d_count, format, mult,
                                                reinterpret_cast<unsigned char*>(rows));
    return cudaGetLastError();
}

}  // namespace m2s
