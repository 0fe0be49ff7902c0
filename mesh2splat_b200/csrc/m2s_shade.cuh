// m2s_shade.cuh — what both conversion kernels use: the per-triangle record the raster kernel leaves for the fragment
// stage, the sampler, the shading of one fragment per layout, and the emission of a warp's 32 staged records.
// The raster kernel (m2s_raster.cu) shades the small triangles of light units itself (direct path); the fragment kernel
// (m2s_fragment.cu) shades everything else.
#pragma once
#include <cstddef>
#include "m2s_codec.cuh"
#include "m2s_device.cuh"
#include "m2s_ptx.cuh"
#include "m2s_span.cuh"

// resident raster warps per SM per raster kind (a multiple of 4: register allocation granularity)
#ifndef M2S_RASTER_WARPS
#define M2S_RASTER_WARPS 16
#endif
#ifndef M2S_RASTER_WARPS_3MAP
#define M2S_RASTER_WARPS_3MAP 16
#endif

namespace m2s {

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

// the exact row spans of a record's candidate box (m2s_span.cuh); h: the box's rows
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

// Appended launches (m2s_convert_host pipelines a scene in triangle chunks): this launch's records follow those of the
// earlier chunks (base); the cap applies to the running index, as the reference's counter does (room: records left).
struct OutRange { unsigned long long base, room; };
__device__ __forceinline__ OutRange out_range(const ConvertArgs& a) {
    unsigned long long base = 0;
    for (uint32_t j = 0; j < a.nprev; ++j) base += *reinterpret_cast<const volatile unsigned long long*>(a.prev_totals + j);
    return {base, a.cap > base ? a.cap - base : 0ull};
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
struct Weights2 {           // filter weights of a footprint pair: bilinear x 1/255 x level blend (1-f, f)
    float2 w00, w10, w01, w11;
};
struct Bilin2 {             // the 2x2 footprints of one map on its two mip levels
    uint32_t i00[2], i10[2], i01[2], i11[2];  // texel indices relative to the level starts
    Weights2 w;
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
    b.w.w00 = fmul2(bx, by); b.w.w10 = fmul2(ax, by); b.w.w01 = fmul2(bx, cy); b.w.w11 = fmul2(ax, cy);
    return b;
}
// The texels of one map's footprints: tx[0..3] = level 0 (00, 10, 01, 11), tx[4..7] = level 1; a map that is not bound
// loads nothing, a single-level lookup (f = 0) loads nothing on level 1.  Returns whether the map is bound.
__device__ __forceinline__ bool fetch_footprint(const uint32_t* __restrict__ texb, const TexRef& ref, float f, const Bilin2& b, uint32_t* tx) {
    const bool has = ref.off0 != 0xffffffffu, two = has && f > 0.0f;
    const uint32_t o0 = has ? ref.off0 : 0u, o1 = ref.off1;  // uniform base + 32-bit texel index
    tx[0] = has ? __ldg(texb + (o0 + b.i00[0])) : 0u; tx[1] = has ? __ldg(texb + (o0 + b.i10[0])) : 0u;
    tx[2] = has ? __ldg(texb + (o0 + b.i01[0])) : 0u; tx[3] = has ? __ldg(texb + (o0 + b.i11[0])) : 0u;
    tx[4] = two ? __ldg(texb + (o1 + b.i00[1])) : 0u; tx[5] = two ? __ldg(texb + (o1 + b.i10[1])) : 0u;
    tx[6] = two ? __ldg(texb + (o1 + b.i01[1])) : 0u; tx[7] = two ? __ldg(texb + (o1 + b.i11[1])) : 0u;
    return has;
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
__device__ __forceinline__ float filt2(const Weights2& w, const uint32_t* tx, uint32_t k4b) {
    float2 acc = fmul2(w.w00, tex_ch2<CH>(tx[0], tx[4], k4b));
    acc = ffma2(w.w10, tex_ch2<CH>(tx[1], tx[5], k4b), acc);
    acc = ffma2(w.w01, tex_ch2<CH>(tx[2], tx[6], k4b), acc);
    acc = ffma2(w.w11, tex_ch2<CH>(tx[3], tx[7], k4b), acc);
    return acc.x + acc.y;
}

// ------------------------------------------------------------------------------------------
// one fragment
// ------------------------------------------------------------------------------------------
// PACKED56 in two halves, so that a warp can have the texel loads of its NEXT 32 fragments in flight while it filters
// and encodes the current ones (direct path of the raster kernel): everything a fragment needs between the halves.
// No texel indices: they would be live across the halves for nothing.
struct Frag1 {
    float Px, Py, Pz, sy;
    Weights2 w;
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
    const float f = tf.frac[0];
    const Bilin2 bl = bilin_setup2(ref, u, v, f2(1.0f - f, f));
    s.w = bl.w;
    s.has = fetch_footprint(texb, ref, f, bl, s.tx);
}
// log_sz: ConvertArgs::log_sz; logtab: kLogfTab or a copy of it (ref_logf)
__device__ __forceinline__ void shade1_finish(float log_sz, const double* logtab, const TriRec<1>& tf, const Frag1& s,
                                              unsigned char* __restrict__ srec_bytes) {
    // converterFS.glsl:55-62,99; parsers.cpp:484-499: SH0, opacity logit, log scale (per triangle)
    const uint32_t k4b = opaque_4b();
    float cr = 1.f, cg = 1.f, cb = 1.f, ca = 1.f;
    if (s.has) { cr = filt2<0>(s.w, s.tx, k4b); cg = filt2<1>(s.w, s.tx, k4b); cb = filt2<2>(s.w, s.tx, k4b); ca = filt2<3>(s.w, s.tx, k4b); }
    const float4 q = *reinterpret_cast<const float4*>(tf.quat), fc = *reinterpret_cast<const float4*>(tf.factor);
    cr *= fc.x; cg *= fc.y; cb *= fc.z; ca *= fc.w;
    float2* s2 = reinterpret_cast<float2*>(srec_bytes);
    s2[0] = make_float2(s.Px, s.Py);
    s2[1] = make_float2(s.Pz, q.x);
    s2[2] = make_float2(q.y, q.z);
    s2[3] = make_float2(q.w, tf.sx);
    s2[4] = make_float2(s.sy, log_sz);
    s2[5] = make_float2(sh0_encode(cr), sh0_encode(cg));
    s2[6] = make_float2(sh0_encode(cb), opacity_logit(ca, logtab));
}
__device__ __forceinline__ void shade1_finish(const ConvertArgs& a, const TriRec<1>& tf, const Frag1& s, unsigned char* __restrict__ srec_bytes) {
    shade1_finish(a.log_sz, kLogfTab, tf, s, srec_bytes);
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
        const float f = tf.frac[m];
        if (m == 0 || !((meta >> m) & 1u)) bl[m] = bilin_setup2(ref, u, vv, f2(1.0f - f, f));
        else bl[m] = bl[0];  // same level sizes and blend as map 0: same footprint and weights
        has[m] = fetch_footprint(texb, ref, f, bl[m], tx[m]);
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
        cr = filt2<0>(bl[0].w, tx[0], k4b); cg = filt2<1>(bl[0].w, tx[0], k4b); cb = filt2<2>(bl[0].w, tx[0], k4b); ca = filt2<3>(bl[0].w, tx[0], k4b);
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
        const float mx = filt2<0>(bl[MN].w, tx[MN], k4b), my = filt2<1>(bl[MN].w, tx[MN], k4b), mz = filt2<2>(bl[MN].w, tx[MN], k4b);
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
        rough = filt2<1>(bl[MM].w, tx[MM], k4b);
        metal = filt2<2>(bl[MM].w, tx[MM], k4b);
    }
    if constexpr (LAYOUT == 0) {
        float4* s4 = reinterpret_cast<float4*>(srec_bytes);
        s4[0] = make_float4(Px, Py, Pz, 1.0f);
        s4[1] = make_float4(cr, cg, cb, ca);
        s4[2] = make_float4(tf.sx, tf.sy, 1e-7f, 0.0f);
        s4[3] = make_float4(nx, ny, nz, 0.0f);
        s4[4] = make_float4(tf.quat[0], tf.quat[1], tf.quat[2], tf.quat[3]);
        s4[5] = make_float4(metal, rough, 0.0f, 1.0f);
    } else {   // the .ply rows; the compressed row's third log scale is log(min(sx,sy) * mult): log is monotonic
        ply_row<LAYOUT - 2>(srec_bytes, make_float3(Px, Py, Pz), make_float3(nx, ny, nz), make_float4(cr, cg, cb, ca),
                            tf.quat, &tf.sx, LAYOUT == 4 ? fminf(tf.sx, tf.sy) : a.log_sz, metal, rough);
    }
    }   // three-map layouts
}

// ------------------------------------------------------------------------------------------
// a warp's 32 staged records -> the output
// ------------------------------------------------------------------------------------------
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

// copy_span for strides that are 8 mod 16, issued by ONE lane: the 16-byte body as one bulk async copy (cp.async.bulk,
// SASS UBLKCP), the 8-byte head and tail as plain stores.  The caller fences the stage's generic-proxy writes
// (fence_proxy_async) before, commits the bulk group after (tma_store_commit; an empty group when nothing was copied), and
// waits for the copy's reads (tma_store_wait_read) before the stage is written again.
template <int STRIDE>
__device__ __forceinline__ void bulk_span(uint8_t* dstbase, unsigned long long boff, const unsigned char* stage, uint32_t nbytes) {
    static_assert(STRIDE % 16 == 8, "the stage shift aligns source and destination of 8-mod-16 strides only");
    if (nbytes == 0) return;
    const uint32_t head = (uint32_t)(boff & 8ull);   // == stage_shift of the first record
    stage += head;
    if (head) *reinterpret_cast<float2*>(dstbase + boff) = *reinterpret_cast<const float2*>(stage);
    const uint32_t body = (nbytes - head) & ~15u;
    if (body) tma_store_1d(dstbase + boff + head, stage + head, body);
    const uint32_t pos = head + body;
    if (pos < nbytes) *reinterpret_cast<float2*>(dstbase + boff + pos) = *reinterpret_cast<const float2*>(stage + pos);
}

// fragment identity: global triangle << 24 | y << 12 | x (meta: the triangle's box origin, TriRec::meta)
__device__ __forceinline__ unsigned long long fragment_key(uint32_t tri, unsigned meta, uint32_t dx, uint32_t dy) {
    return ((unsigned long long)tri << 24) | ((unsigned long long)(((meta >> 16) & 0xfffu) + dy) << 12) |
           (unsigned long long)(((meta >> 4) & 0xfffu) + dx);
}

// The warp's `nfr` staged records are the launch's records [idx, idx + nfr): the ones below `room` go to the output —
// the local buffer at base + idx, or (gather: the fused multi-GPU gather) every rank's final buffer at goff + idx, clipped
// at the final buffers' capacity — and lane l of those writes key(), the key of its fragment, when keys are wanted.
// rot: where the rotation over the destinations starts.
template <int STRIDE, class Key>
__device__ __forceinline__ void emit_records(const ConvertArgs& a, const unsigned char* stage, uint32_t nfr, unsigned long long idx,
                                             unsigned long long base, unsigned long long room, bool gather, unsigned long long goff,
                                             uint32_t rot, Key key, int lane) {
    uint32_t nval = 0;
    if (idx < room) nval = (uint32_t)min((unsigned long long)nfr, room - idx);
    if (!gather) {
        copy_span<STRIDE>(a.out, (base + idx) * (unsigned long long)STRIDE, stage, nval * STRIDE, lane);
    } else {
        const unsigned long long gbase = goff + idx;
        uint32_t gval = 0;
        if (gbase < a.gcap) gval = (uint32_t)min((unsigned long long)nval, a.gcap - gbase);
        // destinations are visited in a rotated order (by rank and by span) so that at any moment the grid's stores are
        // spread over all peers' ingress ports instead of converging on peer 0
        uint32_t p = (a.rank + 1u + rot) % a.world;
        for (uint32_t i = 0; i < a.world; ++i) {
            copy_span<STRIDE>(a.peer_out[p], gbase * (unsigned long long)STRIDE, stage, gval * STRIDE, lane);
            p = p + 1 == a.world ? 0 : p + 1;
        }
    }
    if (a.keys != nullptr && (uint32_t)lane < nval) a.keys[base + idx + lane] = key();
}

}  // namespace m2s
