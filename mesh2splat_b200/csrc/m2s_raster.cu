// m2s_raster.cu — the conversion's first kernel: per-TRIANGLE work, set-up and COUNTING.
//
// The two kernels on one stream (this one, then fragment_kernel in m2s_fragment.cu, launched with programmatic dependent
// launch) replace the reference's geometry shader, fixed-function rasteriser, fragment shader and SSBO atomic append
// (converter{GS,FS}.glsl, ConversionPass.cpp:114-116).  What crosses between them is small and stays in the 50 MB L2:
// one 176-192 B record per triangle, 288 B per queued work item — never anything per fragment.
//
// raster_kernel (persistent, one CTA per SM, every warp an autonomous pipeline; one __syncthreads after the descriptor
// tables are copied to shared memory, none in the steady state)
//   work unit = <= 32 consecutive triangles; a warp's first unit is static (global warp id), further ones are
//     claimed from a global counter; the next unit's triangles are in flight (TMA) while this one is processed.
//     Launches of 16-triangle units (ConvertPlan::pair_first): the first pass sets up units 2g and 2g + 1 on the two
//     half warps.  A pass's direct shading is shared with the CTA's other warps (CtaQueue)
//   TMA (cp.async.bulk + mbarrier complete_tx) stages the unit's 144 B/triangle into shared memory (PACKED56 on a scene
//     uploaded whole: 64 B/triangle, only the positions and uvs the set-up reads)
//   per-triangle stage, one LANE per triangle (converterGS.glsl:326-443): longest edge, face normal, dominant
//     axis, orthographic uv, quaternion, UV->3D Jacobian scale; rasteriser set-up: 24.8 fixed-point window
//     coords, int64 edge functions, top-left ownership bits, candidate pixel box (clamped to the call's
//     pixel-row band); the triangle's resolved sampler state (mip level pair, blend fraction, level offsets)
//   coverage is only COUNTED here:
//     small triangles (box <= 64 pixels, <= 32 rows, int32-safe): lane-per-triangle lock-step walk of the box
//       with incremental edge functions (box_mask, m2s_span.cuh) -> 64-bit coverage mask, stored in the record; a warp scan gives every
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
//     shaded by the warp that rasterised them, straight from the records in its shared-memory slice (direct_run); each
//     group of 32 records leaves through one bulk async copy
//   SINGLE launches (ConvertPlan::single_launch: the direct path, no larger triangle possible at the density, nothing
//     appended): every unit is direct, no fragment kernel follows, and the grid's last CTA publishes the count
//
// Bit-exactness: every float operation of the per-triangle stage is written with __f*_rn intrinsics in the
// operation order of the oracle (and of GLM, which the reference's GLSL-as-C++ build uses): coverage is
// bit-exact and Scale/Quaternion match converterGS.glsl bit for bit.  Per-fragment values may use FMA
// contraction / fast reciprocals and are compared with a tolerance.
#include <type_traits>
#include "m2s_plane.cuh"
#include "m2s_ptx.cuh"
#include "m2s_shade.cuh"

namespace m2s {

// M2S_TRACE builds: per-warp SUMS over all the warp's units, kTraceWarpSlots slots per raster warp after the trace's
// header (scripts/trace_raster.py).  Phases are clock64() deltas (SM cycles: the globaltimer ticks too coarsely for one
// unit); TR_PHASE adds the cycles since the previous mark to its slot.  The three *Ns slots are absolute globaltimer
// stamps (entry, unit-loop exit, exit) that place the warps' work inside the launch.  Fire-and-forget atomics: the
// trace adds no wait to the chain it measures.
enum TraceSlot {
    kTrLoadWait, kTrSetup, kTrWalkScan, kTrLarger, kTrReserve, kTrList, kTrShade, kTrUnitEnd, kTrTail,
    kTrUnits, kTrDirectUnits, kTrGroups, kTrCycles, kTrNanos, kTrEntry, kTrEntryNs, kTrLoopExitNs, kTrExitNs
};
static_assert(kTrExitNs < kTraceWarpSlots, "trace slots per raster warp");
#ifdef M2S_TRACE
#define TR_SLOT(s) (kTraceHeader + ((size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * kTraceWarpSlots + (s))
#define TR_PHASE(a, s) do { const long long n_ = clock64(); if ((a).trace && (threadIdx.x & 31) == 0) atomicAdd((a).trace + TR_SLOT(s), (unsigned long long)(n_ - tr_prev_)); tr_prev_ = n_; } while (0)
#define TR_ADD(a, s, v) do { if ((a).trace && (threadIdx.x & 31) == 0) atomicAdd((a).trace + TR_SLOT(s), (unsigned long long)(v)); } while (0)
#else
#define TR_PHASE(a, s) do { } while (0)
#define TR_ADD(a, s, v) do { } while (0)
#endif

template <int RK>
struct __align__(128) WarpBlock {
    float4 tri[kUnitTris * 9];                    // 4608 B, TMA destination (the 64-byte stream uses 2048 B of it)
    TriRec<RCfg<RK>::kMaps> rec[kUnitTris];       // TMA source
    BlockRef pend[kStashItems * kItemBlocks];     // the stash: row blocks of up to kStashItems work items
    uint32_t itN[kStashItems];                    // blocks per item | kItUnit / kItSplit
    uint32_t itTotal[kStashItems];                // fragments per item
    uint64_t bar;
    double logtab[RK == 1 ? 32 : 1];              // PACKED56: the direct path's copy of ref_logf's table (kLogfTab)
    uint32_t left;                                // posted pieces of this warp's direct pass not yet shaded (CtaQueue)
};
static_assert(offsetof(WarpBlock<1>, pend) % 16 == 0 && sizeof(WarpBlock<1>::pend) >= kUnitTris * kSlimTriBytes,
              "PACKED56's 144-byte route restages a pass's triangles in their 64-byte form into the stash (restage_slim)");

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
// the CTA's threads copy the tables to `base` when they fit (kTableSmemBytes; the CTA barrier that follows publishes them)
__device__ __forceinline__ Tables copy_tables(const ConvertArgs& a, unsigned char* base) {
    Tables tabs{a.ranges, a.prims, a.texs, a.nranges};
    const uint32_t br = a.nranges * (uint32_t)sizeof(DRange), bp = a.nprims * (uint32_t)sizeof(DPrim), bt = a.ntex * (uint32_t)sizeof(DTexture);
    if (br + bp + bt <= kTableSmemBytes) {  // uniform across the grid
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
    return tabs;
}

// what the raster kernel itself keeps of a triangle after the set-up (registers of the owning lane)
struct TriSetup {
    long long E0[3] = {0, 0, 0};
    int A[3] = {0, 0, 0}, B[3] = {0, 0, 0};
    int w = 1, h = 0;
    unsigned incl = 0;
};

// The vertex values the set-up reads.  The set-up of PACKED56 (kSlim) reads a triangle in the 64-byte form of
// ConvertArgs::tris_slim (4 float4: {P0 u0} {P1 u1} {P2 u2} {v0 v1 v2 0}), the three-map layouts read the 144-byte AoS
// (9 float4: 3 x {pos3 nrm3 tan4 uv2}).  Both hold the same fp32 bits.
struct TriVerts {
    f3 P[3];
    float u[3], v[3];
};
template <bool kSlim>
__device__ __forceinline__ TriVerts tri_verts(const float4* __restrict__ t4) {
    TriVerts tv;
    if constexpr (kSlim) {
        const float4 a = t4[0], b = t4[1], c = t4[2], d = t4[3];
        tv.P[0] = {a.x, a.y, a.z}; tv.P[1] = {b.x, b.y, b.z}; tv.P[2] = {c.x, c.y, c.z};
        tv.u[0] = a.w; tv.u[1] = b.w; tv.u[2] = c.w;
        tv.v[0] = d.x; tv.v[1] = d.y; tv.v[2] = d.z;
    } else {
        const float4 q0 = t4[0], q3 = t4[3], q6 = t4[6];
        const float4 q2 = t4[2], q5 = t4[5], q8 = t4[8];
        tv.P[0] = {q0.x, q0.y, q0.z}; tv.P[1] = {q3.x, q3.y, q3.z}; tv.P[2] = {q6.x, q6.y, q6.z};
        tv.u[0] = q2.z; tv.u[1] = q5.z; tv.u[2] = q8.z;
        tv.v[0] = q2.w; tv.v[1] = q5.w; tv.v[2] = q8.w;
    }
    return tv;
}
// PACKED56 on a scene without the 64-byte stream (partial uploads, m2s_debug_set_slim_off): the lane's staged 144-byte
// triangle `src` is rewritten into the 64-byte form at `dst`, which the set-up then reads: one form for the set-up.  `dst`
// is the lane's slot in a free area of its warp's slice; the lane reads back only what it wrote itself.
__device__ __forceinline__ const float4* restage_slim(const float4* __restrict__ src, float4* __restrict__ dst) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {   // vertex k: position = float4 3k, uv = the upper half of float4 3k + 2
        const float4 p = src[3 * k];
        dst[k] = make_float4(p.x, p.y, p.z, src[3 * k + 2].z);
    }
    dst[3] = make_float4(src[2].w, src[5].w, src[8].w, 0.0f);
    return dst;
}

// ------------------------------------------------------------------------------------------
// per-triangle stage + rasteriser set-up.  t4: the staged triangle in shared memory, in the form tri_verts<RK == 1> reads.
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

    // vertex data: positions and uvs
    const TriVerts tv = tri_verts<RK == 1>(t4);
    const f3 P0 = tv.P[0], P1 = tv.P[1], P2 = tv.P[2];

    // converterGS.glsl:327-397: face frame and orthographic uv (m2s_plane.cuh)
    f3 e1, n;
    float ou[3], ov[3];
    ortho_uv(tv.P, pr, e1, n, ou, ov);

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
        const float* uvx = tv.u;
        const float* uvy = tv.v;
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
        put(0, 4, P0.x, P1.x, P2.x); put(1, 4, P0.y, P1.y, P2.y); put(2, 4, P0.z, P1.z, P2.z);   // position
        put(3, 4, tv.u[0], tv.u[1], tv.u[2]);                                                    // u
        put(12, 1, tv.v[0], tv.v[1], tv.v[2]);                                                   // v
    }

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
// work items of the fragment kernel
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t block_ref(uint32_t slot, uint32_t row_begin, uint32_t nrows) {
    return slot | (row_begin << 5) | (nrows << 17);
}

// A warp collects the work items of its current unit in shared memory (WarpBlock::pend / it*) and publishes them
// with ONE 64-bit atomicAdd that reserves both the output range (low 40 bits: fragments) and the queue slots
// (high 24 bits) — the reference does one atomicCounterIncrement per fragment (converterFS.glsl:46).
struct Stash {                // warp-uniform registers
    uint32_t n_it = 0;        // closed items
    uint32_t cur_nb = 0;      // blocks of the open item
    uint32_t cur_total = 0;   // fragments of the open item
    uint32_t frags = 0;       // fragments of the closed items
    uint32_t slots = 0;       // queue slots of the closed items
    unsigned long long seen = 0;  // a lower bound of the global fragment counter (from this warp's last reservation)
};

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

// The covered pixels of this lane's small triangle (coverage mask `hits` of its w-wide box), listed from list[k] on as
// slot | column << 5 | row << 11 — u32 entries in a micro item, u16 entries for the direct path.
template <class T>
__device__ __forceinline__ void list_pixels(T* list, uint32_t k, unsigned long long hits, uint32_t w, uint32_t slot) {
    const uint32_t inv = (65536u + w - 1u) / w;  // row = bit / w by a 16.16 reciprocal (exact for bit < 64, w <= 64)
    while (hits) {
        const uint32_t b = (uint32_t)__ffsll((long long)hits) - 1u;
        hits &= hits - 1ull;
        const uint32_t row = (b * inv) >> 16, col = b - row * w;
        list[k++] = (T)(slot | (col << 5) | (row << 11));
    }
}

// The full rounds of a direct pass whose list exceeds the slice: this lane's pixels sit at places k.. of the pass's list;
// only those in the window [lo, lo + n) are listed, at place - lo.
__device__ __forceinline__ void list_pixels_window(unsigned short* list, uint32_t k, unsigned long long hits, uint32_t w, uint32_t slot,
                                                   uint32_t lo, uint32_t n) {
    const uint32_t inv = (65536u + w - 1u) / w;
    for (; k < lo && hits; ++k) hits &= hits - 1ull;   // the places before the window
    for (; k < lo + n && hits; ++k) {
        const uint32_t b = (uint32_t)__ffsll((long long)hits) - 1u;
        hits &= hits - 1ull;
        const uint32_t row = (b * inv) >> 16, col = b - row * w;
        list[k - lo] = (unsigned short)(slot | (col << 5) | (row << 11));
    }
}

// the unit's small triangles as one item (blocks implicit: one per triangle, TriRec::first/hits).  A unit with at
// most 32 such fragments (sub-pixel meshes: most units of a 1 M-triangle scan) lists them in the item instead: the
// fragment kernel then needs neither the staged unit nor its span table.  hits/w/first/slot: this lane's triangle.
template <int RK>
__device__ __forceinline__ void stash_unit_item(const ConvertArgs& a, WarpBlock<RK>& wb, uint32_t unit, Stash& st, uint32_t total_small,
                                                uint32_t ntri, unsigned long long hits, uint32_t w, uint32_t first, uint32_t slot, int lane) {
    if (total_small == 0) return;
    // the open item (if any) stays open: closed items occupy the slots below n_it, the open one is written at n_it
    // only when it closes — so insert the unit item by closing the open one first
    stash_close_item<RK>(a, wb, unit, st, lane);
    const bool micro = total_small <= 32;
    if (micro) list_pixels(reinterpret_cast<uint32_t*>(wb.pend + st.n_it * kItemBlocks), first, hits, w, slot);
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

// CTA-local help queue (shared memory): a work unit whose larger triangles add up to many row blocks (a wall of a
// building: 28 triangles x 4 blocks x 2000 fragments) would keep ONE warp busy for hundreds of microseconds while the
// others are done: it posts its tall triangles here, in pieces of kDeferBlocks row blocks, and every warp of the CTA that
// has run out of units takes tickets.  Shared-memory atomics only: a grid-wide queue was tried (r02) and lost to the
// serialisation of same-address global atomics (one per unit / per claim: 8-30 us at 2-30 k units).
// The same queue shares the shading of a direct pass (h < 0, SharePiece): the pieces of kSharePiece listed fragments after
// the owner's first kShareFirst, each shaded by whichever warp of the CTA takes it first: the owner or a warp out of units.
struct SharePiece {
    unsigned long long first;     // output index of the owner's listed fragment 0
    uint32_t owner;               // warp of the CTA whose slice holds the records and the list
    uint32_t tri0;                // the scene triangle of the owner's record 0
    uint32_t f0, f1;              // listed fragments [f0, f1)
};
struct CtaEntry {
    union { RowState rs; SharePiece sp; };   // 64 B
    int h;                        // < 0: a shading piece (sp)
    uint32_t unit, slot, rb0, rb1;
    volatile uint32_t ready;      // written last
    uint32_t taken;               // shading pieces: set by the warp that shades it
    uint32_t pad;
};
// Capacity and piece sizes of a direct pass's sharing: the queue takes the CTA's shared memory up to the 227 KB limit (58
// entries of 88 B).  On the bench scene (H100, 16 warps per CTA, ~300 listed fragments per pass) an owner that keeps 192
// fragments posts 33-45 pieces of 64 per CTA; one that keeps only 64 would post 63-74, the queue would be full before
// the last warps post, and those would keep all their pieces (DESIGN.md section 4)
constexpr uint32_t kCtaQueueCap = 58;
constexpr uint32_t kShareFirst = 6 * 32;   // fragments of a direct pass its owner shades before the posted pieces
constexpr uint32_t kSharePiece = 2 * 32;   // fragments per posted piece
static_assert(kShareFirst % 32 == 0 && kSharePiece % 32 == 0 && 2 * M2S_DIRECT_MAX <= kShareFirst + 32 * kSharePiece,
              "pieces start on a group; one lane posts each piece of a pass");
struct CtaQueue {
    uint32_t tail;                // entries posted (may exceed the capacity: the poster keeps the overflow)
    uint32_t head;                // tickets taken
    uint32_t active;              // warps of the CTA still inside their unit loop
    uint32_t pad;
    CtaEntry q[kCtaQueueCap];
};

// A post of n entries: cta_reserve reserves [base, base + n), the first `fit` of them in the queue (the poster keeps the
// rest); cta_publish fills entry base + i, i < fit, through fill(entry, i) and marks it ready.  Two steps: a direct pass
// sets WarpBlock::left in between.
struct CtaPost {
    uint32_t base, fit;
};
__device__ __forceinline__ CtaPost cta_reserve(CtaQueue& cq, uint32_t n, int lane) {
    uint32_t base = 0;
    if (lane == 0) base = atomicAdd_block(&cq.tail, n);
    base = __shfl_sync(0xffffffffu, base, 0);
    return {base, base < kCtaQueueCap ? min(n, kCtaQueueCap - base) : 0u};
}
template <class Fill>
__device__ __forceinline__ void cta_publish(CtaQueue& cq, uint32_t base, uint32_t fit, int lane, Fill&& fill) {
    if ((uint32_t)lane < fit) {
        CtaEntry& e = cq.q[base + lane];
        fill(e, (uint32_t)lane);
        __threadfence_block();
        e.ready = 1u;
    }
}

// takes the shading piece of entry t unless another warp has: `won` becomes 1 on every lane if this warp took it, else 0
__device__ __forceinline__ void cta_take(CtaQueue& cq, uint32_t t, uint32_t& won, int lane) {
    if (lane == 0) won = atomicExch(&cq.q[t].taken, 1u) == 0u;
    won = __shfl_sync(0xffffffffu, won, 0);
}

// a warp that is out of units waits for the entry of its ticket t: true once the entry is posted and ready, false once no
// warp of the CTA can post it any more
__device__ __forceinline__ bool cta_ticket_wait(CtaQueue& cq, uint32_t t, int lane) {
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
    return __shfl_sync(0xffffffffu, (int)have, 0);
}

// ------------------------------------------------------------------------------------------
// DIRECT path: the fragments of a light unit's small triangles, listed in the unit's shared-memory slice, are shaded
// by the warp that rasterised them, in groups of 32.  Used when the warps have several units each (n_units > resident
// warps: on an H100 (132 SMs x 16 warps x 32 triangles) meshes of > 67 k triangles, where most units emit a handful of
// fragments and a work item + a staged unit per unit would cost more than the shading); with one unit per warp the 16
// warps of an SM are too few to hide the latency of the shading chain and the unit goes to the fragment kernel (that was
// faster than the direct path, also with CTA-level group stealing and software pipelining, when measured during
// development).
// The worker: the listed fragments [f0, f1) of the unit(s) in `src`'s slice, 32 at a time (PACKED56).  Out of line: its
// registers are not the raster loop's.  It takes the few per-launch values it needs as arguments (through a ConvertArgs
// reference every group re-loaded them).  dfirst: the output index of listed fragment 0; tri0: the scene triangle of
// record 0; base / room: OutRange; logtab: ref_logf's table.  `src` is the shading warp's own slice, or another warp's
// for a shared piece (CtaQueue); the stage is always the shading warp's own dead triangle staging area.
// A group's records leave the stage as one bulk async copy issued by lane 0 (bulk_span, with emit_records' capacity cut);
// the groups alternate between the two halves of the stage, so a group is shaded while the previous one's copy reads.
// `par` is the half of the next group; the half after the last group is returned, so that the alternation holds across calls.
// ------------------------------------------------------------------------------------------
__device__ __noinline__ uint32_t direct_run(const WarpBlock<1>& src, uint32_t f0, uint32_t f1, unsigned long long dfirst, uint32_t tri0,
                                            unsigned char* stage0, uint32_t par, uint8_t* out, unsigned long long* keys,
                                            const uint32_t* __restrict__ texb, const double* logtab, float log_sz,
                                            unsigned long long base, unsigned long long room, int lane) {
    constexpr int kStride = Cfg<1>::kStride;
    constexpr uint32_t kHalf = kUnitTris * kTriBytes / 2;
    static_assert(8 + 32 * kStride <= kHalf && kHalf % 16 == 0, "two output stages (32 records + the shift) in the triangle staging area");
    const unsigned short* list = reinterpret_cast<const unsigned short*>(src.pend);
    for (uint32_t g0 = f0; g0 < f1; g0 += 32, par ^= 1u) {
        const uint32_t nfr = min(32u, f1 - g0);
        const uint32_t e = list[g0 + min((uint32_t)lane, nfr - 1u)];  // idle lanes shadow the last fragment
        const uint32_t slot = e & 31u;
        const int dxi = (int)((e >> 5) & 63u), dyi = (int)(e >> 11);
        const unsigned long long idx = dfirst + g0;
        unsigned char* const stage = stage0 + par * kHalf;
        Frag1 s;
        shade1_fetch(src.rec[slot], dxi, dyi, texb, s);
        if (lane == 0) tma_store_wait_read_but_last();   // the copy from this half, two groups ago
        __syncwarp();
        shade1_finish(log_sz, logtab, src.rec[slot], s, stage + stage_shift<kStride>(base + idx) + lane * kStride);
        fence_proxy_async();   // the stage's writes, before the bulk copy reads them
        __syncwarp();
        const uint32_t nval = idx < room ? (uint32_t)min((unsigned long long)nfr, room - idx) : 0u;
        if (lane == 0) {   // one bulk group per group of records, empty past the cut: "two groups ago" stays exact
            bulk_span<kStride>(out, (base + idx) * (unsigned long long)kStride, stage, nval * kStride);
            tma_store_commit();
        }
        if (keys != nullptr && (uint32_t)lane < nval) keys[base + idx + lane] = fragment_key(tri0 + slot, src.rec[slot].meta, (uint32_t)dxi, (uint32_t)dyi);
    }
    return par;
}

// The sharing of a direct pass of `owner`, this warp: the pass's list [0, dsum) is cut into groups of 32 from 0, across
// the boundary of its two units: only the last group can be partial.  This warp shades the first kShareFirst fragments at
// once; the rest goes to the CTA's help queue in pieces of kSharePiece, which this warp then shades in order unless
// another warp has taken them: a warp that is out of units takes the pieces this warp has not reached (the late claim
// cannot balance a pass's weight).  Returns the pieces posted and how many of them this warp shaded itself.
struct DirectShare {
    uint32_t fit, done;
};
// places of a direct pass's list in the slice (the stash area): a pass lists up to this many fragments at once.  It holds
// two units of M2S_DIRECT_MAX, so a pass of the two-kernel route takes one round; only single launches (every unit direct,
// ConvertPlan::single_launch) list and shade a longer pass in rounds
constexpr uint32_t kDirectList = 2 * M2S_DIRECT_MAX;
static_assert(kDirectList * sizeof(unsigned short) <= sizeof(BlockRef) * kStashItems * kItemBlocks, "a round's list fits the stash");
template <class Shade>
__device__ __forceinline__ DirectShare direct_share(CtaQueue& cq, WarpBlock<1>& wb, uint32_t owner, uint32_t dsum, unsigned long long dfirst,
                                                    uint32_t tri0, Shade&& shade, int lane) {
    const uint32_t npiece = dsum > kShareFirst ? (dsum - kShareFirst + kSharePiece - 1) / kSharePiece : 0u;
    CtaPost q{0, 0};
    if (npiece) {
        q = cta_reserve(cq, npiece, lane);
        if (lane == 0) wb.left = q.fit;
        __threadfence_block();   // the count, the records and the list, before the pieces are posted
        __syncwarp();
        cta_publish(cq, q.base, q.fit, lane, [&](CtaEntry& e, uint32_t i) {
            e.h = -1;
            e.sp.first = dfirst; e.sp.owner = owner; e.sp.tri0 = tri0;
            e.sp.f0 = kShareFirst + i * kSharePiece; e.sp.f1 = min(dsum, e.sp.f0 + kSharePiece);
        });
    }
    shade(wb, 0, min(dsum, kShareFirst), dfirst, tri0);
    uint32_t done = 0;
    for (uint32_t p = 0; p < npiece; ++p) {
        uint32_t won = 1;
        if (p < q.fit) {
            cta_take(cq, q.base + p, won, lane);
            done += won;
        }
        const uint32_t f0 = kShareFirst + p * kSharePiece;
        if (won) shade(wb, f0, min(dsum, f0 + kSharePiece), dfirst, tri0);
    }
    return {q.fit, done};
}

// other warps may still read the records and the list of this warp's slice: wait until they have shaded the pieces
// they took, before the slice is rewritten
__device__ __forceinline__ void direct_share_wait(WarpBlock<1>& wb, DirectShare sh, int lane) {
    if (sh.fit) {
        if (lane == 0) {
            if (sh.done) atomicSub_block(&wb.left, sh.done);
            while (*reinterpret_cast<volatile uint32_t*>(&wb.left) != 0u) __nanosleep(32);
            __threadfence_block();
        }
        __syncwarp();
    }
}

// help: tickets on the CTA's queue until no warp of the CTA can post any more.  A tall triangle's row blocks are counted
// into this warp's stash; a shading piece is shaded from its owner's slice of `smem`, unless its owner got there first
template <int RK, class Shade>
__device__ __forceinline__ void help_cta(const ConvertArgs& a, unsigned char* smem, WarpBlock<RK>& wb, Stash& st, CtaQueue& cq,
                                         Shade&& shade, int lane) {
    if (lane == 0) atomicSub_block(&cq.active, 1u);
    for (;;) {
        uint32_t t = 0;
        if (lane == 0) t = atomicAdd_block(&cq.head, 1u);
        t = __shfl_sync(0xffffffffu, t, 0);
        if (t >= kCtaQueueCap) break;  // beyond the capacity nothing is ever posted
        if (!cta_ticket_wait(cq, t, lane)) break;
        const CtaEntry& e = cq.q[t];
        if (e.h < 0) {
            if constexpr (RK == 1) {
                uint32_t won = 0;
                cta_take(cq, t, won, lane);
                if (won) {
                    WarpBlock<RK>& src = *reinterpret_cast<WarpBlock<RK>*>(smem + (size_t)e.sp.owner * sizeof(WarpBlock<RK>));
                    cp_async_wait_all();   // this warp's wb.logtab, if it never shaded a unit of its own
                    __syncwarp();
                    shade(src, e.sp.f0, e.sp.f1, e.sp.first, e.sp.tri0);
                    __syncwarp();
                    if (lane == 0) { __threadfence_block(); atomicSub_block(&src.left, 1u); }   // its slice may be rewritten
                }
            }
            continue;
        }
        const RowState rs = e.rs;
        const int h = e.h;
        const uint32_t eu = e.unit, es = e.slot;
        const int rb0 = (int)e.rb0, rb1 = (int)e.rb1;
        count_blocks<RK>(a, wb, eu, st, rs, h, es, rb0, rb1, lane);
        stash_close_item<RK>(a, wb, eu, st, lane);
        stash_flush<RK>(a, wb, eu, st, lane);
    }
}

// ------------------------------------------------------------------------------------------
// raster_kernel
// ------------------------------------------------------------------------------------------
template <int RK>
__global__ void __launch_bounds__(RCfg<RK>::kWarps * 32, 1) raster_kernel(const __grid_constant__ ConvertArgs a) {
    using C = RCfg<RK>;
    using Rec = TriRec<C::kMaps>;
    extern __shared__ __align__(128) unsigned char smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    WarpBlock<RK>& wb = *reinterpret_cast<WarpBlock<RK>*>(smem + (size_t)warp * sizeof(WarpBlock<RK>));
    constexpr bool kDirectOK = (RK == 1);   // PACKED56: the records carry everything the shading needs
    // PACKED56 stages only the positions and uvs when the scene has them repacked (64 B per triangle instead of 144).  Read
    // from the kernel parameters where it is used: a pointer kept across the unit loop takes registers the loop needs
    auto slim = [&]() { return RK == 1 && a.tris_slim != nullptr; };
    auto tri_size = [&]() { return slim() ? (uint32_t)kSlimTriBytes : (uint32_t)kTriBytes; };
#ifdef M2S_TRACE
    long long tr_prev_ = clock64();
    const long long tr_c0_ = tr_prev_;
    const unsigned long long tr_ns0_ = gtimer_ns();
#endif

    if (lane == 0) {
        mbar_init(&wb.bar, 1);
        fence_barrier_init();
    }
    __syncwarp();
    // the first unit of every warp is static (unit = global warp id): no atomic, and nobody can grab two units
    // while a neighbour gets none.  Paired launches (ConvertPlan::pair_first): the first pass takes units 2g and 2g + 1,
    // one per half warp, on one load
    const uint32_t nwarps_total = gridDim.x * (blockDim.x >> 5);
    const uint32_t gwarp = blockIdx.x + gridDim.x * warp;  // warp w of every CTA before warp w+1 of any: SMs fill evenly
    bool pair = kDirectOK && a.pair_first != 0;
    uint32_t unit = pair ? 2 * gwarp : gwarp;
    const uint32_t claim_base = pair ? 2 * nwarps_total : nwarps_total;   // the first unit the counter hands out
    auto issue_load = [&](uint32_t u, uint32_t n) {  // lane 0 only: up to n triangles from unit u on
        const uint32_t t0 = u * a.unit_tris;
        const uint32_t bytes = min(n, a.tri_count - t0) * tri_size();
        const unsigned char* src = reinterpret_cast<const unsigned char*>(slim() ? a.tris_slim : a.tris);
        fence_proxy_async();
        mbar_arrive_expect_tx(&wb.bar, bytes);
        tma_load_1d(wb.tri, src + ((size_t)a.tri_first + t0) * tri_size(), bytes, &wb.bar);
    };
    auto claim = [&]() { return claim_base + atomicAdd(a.claim, 1u); };   // lane 0 only: the next unit
    // ref_logf's table for the direct path's opacities -> the warp's slice, as an asynchronous copy that lands while the
    // first unit is set up (waited for before the first shading; a CTA-wide copy would wait at the barrier below: ~1 us
    // more per warp, measured on the H100)
    if constexpr (kDirectOK) cp_async_8(wb.logtab + lane, kLogfTab + lane);

    const Tables tabs = copy_tables(a, smem + (size_t)C::kWarps * sizeof(WarpBlock<RK>));
    CtaQueue& cq = *reinterpret_cast<CtaQueue*>(smem + (size_t)C::kWarps * sizeof(WarpBlock<RK>) + kTableSmemBytes);
    if (threadIdx.x == 0) { cq.tail = 0; cq.head = 0; cq.active = blockDim.x >> 5; }
    // re-arm the other scheduler set for the next launch: the launch before this one used it and has ended (no launch of
    // this kernel overlaps the one before it), and the next one starts after this one's last kernel
    if (blockIdx.x == 0 && threadIdx.x == 0) { *a.next_claim = 0; *a.next_counter = 0ull; }
    if (threadIdx.x < kCtaQueueCap) { cq.q[threadIdx.x].ready = 0u; cq.q[threadIdx.x].taken = 0u; }
    __syncthreads();  // tables + help queue: the only CTA-wide barrier before the end of the kernel
    // the first unit's triangles start moving only now: issued before the table copy, the first loads of all the grid's
    // warps (4.3 MB of slim triangles on the bench) reach HBM at once from a cold L2, and the table loads and this barrier
    // queue behind them (DESIGN.md section 4)
    if (lane == 0 && unit < a.n_units) issue_load(unit, pair ? 2 * a.unit_tris : a.unit_tris);
    const OutRange out = out_range(a);   // the direct path's records
    uint32_t phase = 0;
    uint32_t spar = 0;   // the half of this warp's output stage that its next group of direct records goes to
    Stash st;
    // the listed fragments [f0, f1) of the unit(s) in slice `src`, shaded by this warp through its own stage (direct_run)
    auto shade = [&](const WarpBlock<RK>& src, uint32_t f0, uint32_t f1, unsigned long long first, uint32_t tri0) {
        if constexpr (kDirectOK) {
            spar = direct_run(src, f0, f1, first, tri0, reinterpret_cast<unsigned char*>(wb.tri), spar, a.out, a.keys, a.tex_base,
                              wb.logtab, a.log_sz, out.base, out.room, lane);
            TR_ADD(a, kTrGroups, (f1 - f0 + 31) / 32);
        }
    };
    TR_PHASE(a, kTrEntry);

    while (unit < a.n_units) {
        const uint32_t t0 = unit * a.unit_tris;
        const uint32_t ntri = min(pair ? 2 * a.unit_tris : a.unit_tris, a.tri_count - t0);   // triangles of this pass
        const uint32_t nu = pair && ntri > a.unit_tris ? 2u : 1u;                              // units of this pass
        const int sw = pair ? 16 : 32;   // lanes per unit: lane l sets up triangle l of the pass, of unit `unit + l / sw`
        uint32_t next = 0xffffffffu;
        // launches with a direct path and fewer than three units per warp: the next unit is claimed only once this unit's
        // work is known (after its shading for a direct unit).  A direct unit shades anything from 0 to 16 groups of 32
        // fragments; claimed up front, every warp would get its two units whatever they weigh, and the kernel would end with
        // the warps that drew heavy ones.  Claimed late, a warp that is still shading leaves the remaining units to the
        // warps that are done.  The late claim costs one exposed atomic round trip per unit: with more units per warp the
        // weights average out and the claim stays up front.  The host decides (ConvertPlan::claim_late).
        const bool claim_late = kDirectOK && a.claim_late != 0;
        if (lane == 0) {
            if (a.n_units > nwarps_total && !claim_late) next = claim();  // needed only after the set-up
            tma_store_wait_read();  // the previous unit's record store has finished reading wb.rec
        }
        mbar_wait(&wb.bar, phase);
        phase ^= 1;
        __syncwarp();
        TR_PHASE(a, kTrLoadWait);
        TR_ADD(a, kTrUnits, nu);

        // ---- per-triangle stage: one lane per triangle ----
        uint32_t cnt = 0;
        TriSetup ts;
        Rec& myrec = wb.rec[lane];
        // the staged triangle in the form the set-up reads; the 144-byte route of PACKED56 restages it into the stash, which
        // is empty between passes (stash_flush) and is not written before the set-up is done
        const float4* tri4 = wb.tri + lane * (RK == 1 ? 4 : 9);
        if (RK == 1 && !slim() && (uint32_t)lane < ntri) tri4 = restage_slim(wb.tri + lane * 9, reinterpret_cast<float4*>(wb.pend) + lane * 4);
        if ((uint32_t)lane < ntri) cnt = setup_triangle<RK>(tri4, a.tri_first + t0 + lane, a, tabs, ts, myrec);
        __syncwarp();
        TR_PHASE(a, kTrSetup);
        next = __shfl_sync(0xffffffffu, next, 0);

        // ---- small triangles: lane-per-triangle lock-step walk of the candidate box -> coverage mask ----
        int e0 = 0, e1 = 0, e2 = 0, a0 = 0, a1 = 0, a2 = 0, b0 = 0, b1 = 0, b2 = 0, w = 1;
        bool small = false;
        if (cnt) {
            w = ts.w;
            const int h = ts.h;
            a0 = ts.A[0]; a1 = ts.A[1]; a2 = ts.A[2];
            b0 = ts.B[0]; b1 = ts.B[1]; b2 = ts.B[2];
            // E at the box origin, with the ownership bias folded in: inside <=> all E' >= 0
            const long long E0 = ts.E0[0] - ((ts.incl & 1u) ? 0 : 1);
            const long long E1 = ts.E0[1] - ((ts.incl & 2u) ? 0 : 1);
            const long long E2 = ts.E0[2] - ((ts.incl & 4u) ? 0 : 1);
            const long long lim = 0x7fffffffll;
            const long long s0 = llabs(E0) + (long long)(w - 1) * abs(a0) + (long long)(h - 1) * abs(b0);
            const long long s1 = llabs(E1) + (long long)(w - 1) * abs(a1) + (long long)(h - 1) * abs(b1);
            const long long s2 = llabs(E2) + (long long)(w - 1) * abs(a2) + (long long)(h - 1) * abs(b2);
            small = cnt <= kSmallCand && h <= 32 && s0 < lim && s1 < lim && s2 < lim;
            if (small) { e0 = (int)E0; e1 = (int)E1; e2 = (int)E2; }
        }
        const uint32_t mine = small ? cnt : 0u;
        const unsigned long long hits = box_mask(e0, e1, e2, a0, a1, a2, b0, b1, b2, w, mine, __reduce_max_sync(0xffffffffu, mine));
        const uint32_t nh = (uint32_t)__popcll(hits);
        // the scans run over the lanes of one unit: TriRec::first is relative to the triangle's own unit
        const uint32_t incl_scan = warp_inclusive_scan(nh, lane, sw);
        const uint32_t tot0 = __shfl_sync(0xffffffffu, incl_scan, sw - 1);   // small-triangle fragments of the first unit
        const uint32_t tot1 = __shfl_sync(0xffffffffu, incl_scan, 31);       // ... and of the second (paired pass)
        const uint32_t myrows = small ? (uint32_t)ts.h : 0u;  // rows this triangle contributes to the unit item's span table
        const uint32_t rows_scan = warp_inclusive_scan(myrows, lane, sw);
        if ((uint32_t)lane < ntri) {
            myrec.hits = hits;
            myrec.first = (incl_scan - nh) | ((rows_scan - myrows) << 16);
            myrec.box = cnt ? ((unsigned)ts.w | ((unsigned)ts.h << 13) | (ts.incl << 26) | (small ? kBoxSmall : 0u)) : 0u;
        }
        __syncwarp();
        TR_PHASE(a, kTrWalkScan);
        // DIRECT path (REF96 / PACKED56, single GPU): when a unit's small triangles emit at most M2S_DIRECT_MAX fragments
        // this warp shades them itself, straight from the records in its shared-memory slice — no work item, no record
        // round trip through L2, no second kernel on the critical path.  The triangle staging area (dead since the set-up)
        // is the warp's output stage then, so the next unit's triangles start flying in after the shading instead of now.
        // A single launch has no fragment kernel behind it: every unit is direct, however heavy
        const bool direct_ok = kDirectOK && a.direct_ok != 0;
        const uint32_t dmax = a.single_launch ? 0xffffffffu : (uint32_t)M2S_DIRECT_MAX;
        const bool direct0 = direct_ok && tot0 != 0 && tot0 <= dmax;
        const bool direct1 = nu == 2 && direct_ok && tot1 != 0 && tot1 <= dmax;
        const bool direct = direct0 || direct1;
        const uint32_t hf = (uint32_t)lane / (uint32_t)sw;                 // this lane's unit of the pass
        const unsigned hmask = sw == 32 ? 0xffffffffu : 0xffffu << (hf * 16);   // the lanes of that unit
        const bool my_direct = hf ? direct1 : direct0;
        const uint32_t dfr0 = direct0 ? tot0 : 0u, dsum = dfr0 + (direct1 ? tot1 : 0u);   // the pass's list: unit 0's, then unit 1's
        auto claim_now = [&]() {   // the next unit, claimed once this one's work is known
            if (lane == 0) next = claim();
            next = __shfl_sync(0xffffffffu, next, 0);
        };
        if (claim_late && !direct) claim_now();
        if (!direct && lane == 0 && next < a.n_units) issue_load(next, a.unit_tris);

        // ---- all other triangles: the warp counts one triangle at a time, one lane per pixel row; the tall triangles of
        // a heavy unit are posted to the CTA's help queue instead (see CtaQueue).  Every work item names one unit, so the
        // first unit of a paired pass reserves its items before the second unit's are stashed ----
        const bool larger = cnt != 0 && !small;
        const uint32_t gm_all = __ballot_sync(0xffffffffu, larger);
        const uint32_t myblocks = larger ? (uint32_t)(ts.h + 31) / 32u : 0u;
        for (uint32_t k = 0; k < nu; ++k) {
            const uint32_t u = unit + k, lo = k * (uint32_t)sw;
            const unsigned umask = nu == 1 ? 0xffffffffu : 0xffffu << lo;
            const bool in_u = (umask >> lane) & 1u;
            const uint32_t unit_blocks = __reduce_add_sync(0xffffffffu, in_u ? myblocks : 0u);
            unsigned gm = gm_all & umask;
            if (unit_blocks > kDeferUnitBlocks) {
                unsigned dm = __ballot_sync(0xffffffffu, myblocks >= 2) & umask;
                while (dm) {
                    const int s = __ffs(dm) - 1;
                    dm &= dm - 1;
                    int h;
                    const RowState rs = row_state(wb.rec[s], h);
                    const uint32_t nb = (uint32_t)(h + 31) / 32u, nent = (nb + kDeferBlocks - 1) / kDeferBlocks;
                    const CtaPost q = cta_reserve(cq, nent, lane);   // the first q.fit pieces go to the queue
                    cta_publish(cq, q.base, q.fit, lane, [&](CtaEntry& e, uint32_t i) {
                        e.rs = rs; e.h = h; e.unit = u; e.slot = (uint32_t)s - lo;
                        e.rb0 = i * kDeferBlocks; e.rb1 = min(nb, (i + 1) * kDeferBlocks);
                    });
                    if (q.fit < nent) count_blocks<RK>(a, wb, u, st, rs, h, (uint32_t)s - lo, (int)(q.fit * kDeferBlocks), 1 << 20, lane);  // the rest stays here
                    gm &= ~(1u << s);
                }
            }
            while (gm) {
                const int s = __ffs(gm) - 1;
                gm &= gm - 1;
                int h;
                const RowState rs = row_state(wb.rec[s], h);  // broadcast reads of the record
                count_blocks<RK>(a, wb, u, st, rs, h, (uint32_t)s - lo, 0, 1 << 20, lane);
            }
            stash_close_item<RK>(a, wb, u, st, lane);
            if (!(k ? direct1 : direct0))
                stash_unit_item<RK>(a, wb, u, st, k ? tot1 : tot0, k ? ntri - lo : min(ntri, (uint32_t)sw), in_u ? hits : 0ull,
                                    (uint32_t)w, incl_scan - nh, (uint32_t)lane - lo, lane);
            if (k + 1 < nu) stash_flush<RK>(a, wb, u, st, lane);
        }
        TR_PHASE(a, kTrLarger);
        // ONE atomicAdd per pass (unless the stash filled up on the way, or both units of a pair queue items) reserves the
        // output range and the queue slots of everything the pass emits; the direct fragments come last
        const unsigned long long dfirst = stash_flush<RK>(a, wb, unit + nu - 1, st, lane, dsum);   // the stash area is free after this
        TR_PHASE(a, kTrReserve);
        if constexpr (kDirectOK) {
            if (direct) {
                TR_ADD(a, kTrDirectUnits, (direct0 ? 1 : 0) + (direct1 ? 1 : 0));
                // every lane of a direct unit lists the covered pixels of its triangle at their place in the pass's list.  A
                // list longer than the slice's kDirectList places (single launches only) goes in rounds: the full rounds first,
                // each shaded before the next rewrites the list, then the rest as a pass of its own
                uint32_t my0 = (hf ? dfr0 : 0u) + incl_scan - nh;
                unsigned long long my_hits = my_direct ? hits : 0ull;
                uint32_t r0 = 0;
                if (dsum > kDirectList) {
                    cp_async_wait_all();
                    for (; dsum - r0 > kDirectList; r0 += kDirectList) {
                        list_pixels_window(reinterpret_cast<unsigned short*>(wb.pend), my0, my_hits, (uint32_t)w, (uint32_t)lane, r0, kDirectList);
                        __syncwarp();
                        direct_share_wait(wb, direct_share(cq, wb, (uint32_t)warp, kDirectList, dfirst + r0, a.tri_first + t0, shade, lane), lane);
                    }
                    for (; my0 < r0 && my_hits; ++my0) my_hits &= my_hits - 1ull;   // the places listed already
                    my0 = my0 >= r0 ? my0 - r0 : 0u;
                }
                list_pixels(reinterpret_cast<unsigned short*>(wb.pend), my0, my_hits, (uint32_t)w, (uint32_t)lane);
                cp_async_wait_all();   // wb.logtab has landed (a no-op after the first direct unit)
                __syncwarp();
                TR_PHASE(a, kTrList);
                const DirectShare sh = direct_share(cq, wb, (uint32_t)warp, dsum - r0, dfirst + r0, a.tri_first + t0, shade, lane);
                TR_PHASE(a, kTrShade);
                // the stage was written through the generic proxy: every writer fences before the TMA engine writes there again
                fence_proxy_async();
                __syncwarp();
                if (claim_late) claim_now();
                if (lane == 0) tma_store_wait_read();   // the last groups' copies have read the stage
                if (lane == 0 && next < a.n_units) issue_load(next, a.unit_tris);
                direct_share_wait(wb, sh, lane);
            }
        }

        // ---- the pass's records go to global memory for the fragment kernel: one TMA bulk store straight out of
        // this warp's shared-memory slice (every writer fences its generic-proxy writes, then the barrier).  A fully
        // direct unit leaves nothing for the fragment kernel ----
        const bool any = __any_sync(0xffffffffu, cnt != 0 && (!my_direct || (gm_all & hmask) != 0));
        if (any) {
            fence_proxy_async();
            __syncwarp();
            if (lane == 0) {
                tma_store_1d(a.tri_frag + (size_t)t0 * sizeof(Rec), wb.rec, ntri * (uint32_t)sizeof(Rec));
                tma_store_commit();
            }
        }
        unit = next;
        pair = false;
        TR_PHASE(a, kTrUnitEnd);
    }
#ifdef M2S_TRACE
    const unsigned long long tr_loop_ns_ = gtimer_ns();
#endif
    // direct-path launches let the fragment grid launch now: its CTAs take the SMs as the raster CTAs exit and wait there
    // (griddepcontrol.wait) until this grid has completed, instead of being launched and placed after the last exit.
    // Every warp triggers once it is out of units, so the launch fires near the end of the slowest CTA's work; triggered at
    // the kernel's start it made the raster warps slower.  Launches whose fragments the fragment kernel shades (REF96,
    // the .ply rows, single-round launches) keep the launch at the grid's end: REF96 measured slower with it (DESIGN.md section 4)
    if (kDirectOK && a.direct_ok) pdl_launch_dependents();
    help_cta<RK>(a, smem, wb, st, cq, shade, lane);
    // two-kernel launches: no CTA barrier and no grid-wide count at the end: each warp exits once its own bulk stores are
    // complete.  A warp that shades from another warp's slice is done before the help queue lets that slice be rewritten,
    // and shared memory lives until the CTA ends.  The fragment kernel reads the count once this grid has ended
    // (griddepcontrol.wait)
    if (lane == 0) tma_store_wait_all();  // record stores are complete (not just read) before the kernel ends
    if constexpr (kDirectOK) cp_async_wait_all();   // a warp without a direct unit never waited for its wb.logtab
    if constexpr (kDirectOK) {
        if (a.single_launch) {
            // single launches: the grid's last CTA publishes the count.  The queue half of the packed counter stays 0 on
            // these launches (no work item), so it counts the CTAs that are done: one acq_rel add of 1 << 40 per CTA.
            // Every reservation of the CTA precedes its add: the reservations are atomics on the same word, made by the
            // warps before the CTA barrier below, and the barrier orders them before thread 0's add, whose release is
            // cumulative; same-word atomics are totally ordered, so the add that finds gridDim.x - 1 CTAs before it comes
            // after every CTA's every reservation, and the low 40 bits it returns are the final, uncapped count
            __syncthreads();
            if (threadIdx.x == 0) {
                const unsigned long long old = atom_add_acq_rel_gpu(a.counter, 1ull << 40);
                if ((uint32_t)(old >> 40) == gridDim.x - 1) {
                    *a.total_out = old & kFragMask;
#ifdef M2S_TRACE
                    if (a.trace) atomicMax(a.trace + kTrFragEndNs, gtimer_ns());   // the step's end, as the trace places it
#endif
                }
            }
        }
    }
#ifdef M2S_TRACE
    TR_PHASE(a, kTrTail);
    TR_ADD(a, kTrCycles, clock64() - tr_c0_);   // with kTrNanos: the SM clock the cycles convert at
    const unsigned long long tr_exit_ns_ = gtimer_ns();
    TR_ADD(a, kTrNanos, tr_exit_ns_ - tr_ns0_);
    TR_ADD(a, kTrEntryNs, tr_ns0_);
    TR_ADD(a, kTrLoopExitNs, tr_loop_ns_);
    TR_ADD(a, kTrExitNs, tr_exit_ns_);
#endif
}

// ------------------------------------------------------------------------------------------
// host side, declared in m2s_device.cuh
// ------------------------------------------------------------------------------------------
// f(std::integral_constant<int, RK>) for the raster kind of `layout`: REF96, PACKED56, the .ply rows
template <class F>
static auto with_raster_kind(int layout, F&& f) {
    if (layout == 0) return f(std::integral_constant<int, 0>{});
    if (layout == 1) return f(std::integral_constant<int, 1>{});
    return f(std::integral_constant<int, 2>{});
}
template <int RK>
constexpr size_t raster_smem_bytes() { return sizeof(WarpBlock<RK>) * RCfg<RK>::kWarps + kTableSmemBytes + sizeof(CtaQueue); }
static_assert(raster_smem_bytes<0>() <= 232448 && raster_smem_bytes<1>() <= 232448 && raster_smem_bytes<2>() <= 232448,
              "raster kernel: 227 KB of shared memory per CTA");

int convert_warps_per_cta(int layout) {
    return with_raster_kind(layout, [](auto rk) { return RCfg<rk>::kWarps; });
}
size_t tri_frag_bytes(int layout) {
    return with_raster_kind(layout, [](auto rk) { return sizeof(TriRec<RCfg<rk>::kMaps>); });
}

cudaError_t raster_configure(int layout, int* blocks_per_sm) {
    return with_raster_kind(layout, [&](auto rk) {
        const size_t smem = raster_smem_bytes<rk>();
        cudaError_t e = cudaFuncSetAttribute(raster_kernel<rk>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        return cudaOccupancyMaxActiveBlocksPerMultiprocessor(blocks_per_sm, raster_kernel<rk>, RCfg<rk>::kWarps * 32, smem);
    });
}

cudaError_t raster_launch(int layout, const ConvertArgs& args, int grid, cudaStream_t stream) {
    return with_raster_kind(layout, [&](auto rk) {
        raster_kernel<rk><<<grid, RCfg<rk>::kWarps * 32, raster_smem_bytes<rk>(), stream>>>(args);
        return cudaGetLastError();
    });
}

}  // namespace m2s
