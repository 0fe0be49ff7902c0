// m2s_clip.cuh — the clip-space stage the mesh passes share: the mesh depth pre-pass (m2s_depth.cu) and the mesh G-buffer
// pass (m2s_mesh.cu).  GLM's mat4 * vec4 (also the light prepass's, m2s_light.cu), the triangle -> primitive lookup,
// Sutherland-Hodgman against the six planes (z against +-w, x and y against a guard band of +-kClipGuard w), the fan of
// the clipped polygon with the rasteriser's snap and edge set-up (m2s_tile.cuh), the binners' visit of a source
// triangle's fan, and the tile kernels' staging and depth test of a fan triangle (DESIGN §2).  Every operation is
// round-to-nearest fp32 / fp64 with no contraction, so the oracles restate it bit for bit.
//
// The clipper is a template over the polygon vertex: a bare float4 (the depth pass) or a ClipVert, which carries each
// vertex's barycentric weights with respect to its source triangle through the cuts (the G-buffer pass interpolates its
// varyings from them).  Both clip the positions with the same operations, so their polygons are the same.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "m2s_device.cuh"
#include "m2s_tile.cuh"

namespace m2s {

constexpr int kClipMaxPoly = 9;                    // a triangle clipped by six planes keeps at most 3 + 6 vertices
constexpr float kClipGuard = 2.0f;                 // x, y clipped to +-G w: |xw| <= 1.5 * 4096 < 8192 (DESIGN §2)

// GLM mat4 * vec4(x, y, z, w), column-major m: (m0 x + m1 y) + (m2 z + m3 w)
__device__ __forceinline__ float clip_row(const float* m, int row, float x, float y, float z, float w) {
    return ad(ad(ml(m[row], x), ml(m[4 + row], y)), ad(ml(m[8 + row], z), ml(m[12 + row], w)));
}

// the range of triangle `tri` among the n sorted, disjoint primitive ranges; false: the triangle has no primitive
__device__ __forceinline__ bool prim_range(const DRange* ranges, uint32_t n, uint32_t tri, DRange& out) {
    int lo = 0, hi = (int)n - 1;
    while (lo <= hi) {
        const int mid = (lo + hi) >> 1;
        const DRange r = ranges[mid];
        if (tri < r.first) hi = mid - 1;
        else if (tri >= r.end) lo = mid + 1;
        else { out = r; return true; }
    }
    return false;
}

// a polygon vertex with its source-triangle barycentrics
struct ClipVert {
    float4 p;
    float b[3];
};
__device__ __forceinline__ const float4& clip_pos(const float4& v) { return v; }
__device__ __forceinline__ const float4& clip_pos(const ClipVert& v) { return v.p; }
__device__ __forceinline__ float clip_lerp1(float a, float b, float t) { return __fadd_rn(a, __fmul_rn(t, __fsub_rn(b, a))); }
__device__ __forceinline__ float4 clip_lerp(const float4& a, const float4& b, float t) {
    return make_float4(clip_lerp1(a.x, b.x, t), clip_lerp1(a.y, b.y, t), clip_lerp1(a.z, b.z, t), clip_lerp1(a.w, b.w, t));
}
__device__ __forceinline__ ClipVert clip_lerp(const ClipVert& a, const ClipVert& b, float t) {
    ClipVert r;
    r.p = clip_lerp(a.p, b.p, t);
#pragma unroll
    for (int j = 0; j < 3; ++j) r.b[j] = clip_lerp1(a.b[j], b.b[j], t);
    return r;
}

// signed distance to clip plane p (inside iff >= 0): z >= -w, z <= w, x >= -G w, x <= G w, y >= -G w, y <= G w
__device__ __forceinline__ float clip_plane(const float4& v, int p) {
    const float gw = __fmul_rn(kClipGuard, v.w);
    switch (p) {
        case 0: return __fadd_rn(v.z, v.w);
        case 1: return __fsub_rn(v.w, v.z);
        case 2: return __fadd_rn(v.x, gw);
        case 3: return __fsub_rn(gw, v.x);
        case 4: return __fadd_rn(v.y, gw);
        default: return __fsub_rn(gw, v.y);
    }
}

// the point where edge (a inside, b outside) meets the plane, always computed from the inside vertex
template <typename V>
__device__ __forceinline__ V clip_cut(const V& a, const V& b, float da, float db) {
    return clip_lerp(a, b, __fdiv_rn(da, __fsub_rn(da, db)));
}

// The clip-space polygon of the triangle v[0..2] after Sutherland-Hodgman against the six planes in order; returns its
// vertex count (0: nothing left, or a coordinate of v[0..2] is not finite).  A polygon that would grow past kClipMaxPoly
// vertices (only through rounding) keeps its first kClipMaxPoly.
template <typename V>
__device__ int clip_poly(V (&v)[kClipMaxPoly]) {
    bool finite = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float4& p = clip_pos(v[k]);
        finite &= isfinite(p.x) && isfinite(p.y) && isfinite(p.z) && isfinite(p.w);
    }
    if (!finite) return 0;
    bool inside = true;
#pragma unroll
    for (int p = 0; p < 6; ++p)
#pragma unroll
        for (int k = 0; k < 3; ++k) inside &= clip_plane(clip_pos(v[k]), p) >= 0.0f;
    if (inside) return 3;
    int n = 3;
    for (int p = 0; p < 6 && n > 0; ++p) {
        V o[kClipMaxPoly];
        int m = 0;
        float dp = clip_plane(clip_pos(v[n - 1]), p);
        for (int i = 0; i < n; ++i) {
            const float dc = clip_plane(clip_pos(v[i]), p);
            const int prev = i == 0 ? n - 1 : i - 1;
            if (dc >= 0.0f) {
                if (dp < 0.0f && m < kClipMaxPoly) o[m++] = clip_cut(v[i], v[prev], dc, dp);
                if (m < kClipMaxPoly) o[m++] = v[i];
            } else if (dp >= 0.0f && m < kClipMaxPoly) {
                o[m++] = clip_cut(v[prev], v[i], dp, dc);
            }
            dp = dc;
        }
        for (int i = 0; i < m; ++i) v[i] = o[i];
        n = m;
    }
    return n;
}

// the triangle's three vertices as a polygon: set(v[k], clip position, k)
__device__ __forceinline__ void clip_set(float4& v, const float4& c, int) { v = c; }
__device__ __forceinline__ void clip_set(ClipVert& v, const float4& c, int k) {
    v.p = c;
#pragma unroll
    for (int j = 0; j < 3; ++j) v.b[j] = j == k ? 1.0f : 0.0f;
}

// the clip-space polygon of source triangle `tri` of a triangle soup (9 float4 per triangle, m2s_device.cuh), each
// vertex position through the pass's vertex transform xf(x, y, z) -> clip float4; returns its vertex count
template <typename V, typename Xf>
__device__ __forceinline__ int clip_tri_poly(const float4* tris, uint32_t tri, Xf&& xf, V (&v)[kClipMaxPoly]) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float4 p = __ldg(tris + (size_t)tri * 9 + k * 3);
        clip_set(v[k], xf(p.x, p.y, p.z), k);
    }
    return clip_poly(v);
}

struct FanTri {
    TileTri t;
    float z[3];   // window depth (z / w) 0.5 + 0.5 of the three vertices
};

// fan triangle (v0, vk+1, vk+2) of a W x H viewport: perspective divide, the viewport transform, snap and edge set-up.
// kCull: a triangle whose snapped window-space area is negative (clockwise, y up) is set up empty, as a zero area always
// is (GL_CULL_FACE with glCullFace(GL_BACK), glFrontFace(GL_CCW)).
template <bool kCull, typename V>
__device__ __forceinline__ void clip_fan(const V (&v)[kClipMaxPoly], int k, uint32_t width, uint32_t height, FanTri& d) {
    const float hw = ml((float)width, 0.5f), hh = ml((float)height, 0.5f);
    int X[3], Y[3];
    bool ok = true;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float4& p = clip_pos(v[c == 0 ? 0 : k + c]);
        bool okc;
        tile_snap(dv(p.x, p.w), dv(p.y, p.w), hw, hh, okc, X[c], Y[c]);
        ok &= okc;
        d.z[c] = ad(ml(dv(p.z, p.w), 0.5f), 0.5f);
    }
    if (kCull && ok) ok = (long long)(X[1] - X[0]) * (Y[2] - Y[0]) - (long long)(X[2] - X[0]) * (Y[1] - Y[0]) >= 0;
    tile_tri_setup(X, Y, ok, (int)width, (int)height, d.t);
}

// the binners' visit of source triangle `tri` (m2s_bin.cuh): unless keep(tri) is false, its clip-space polygon
// (clip_tri_poly with the pass's transform xf) and one pair f(tile, tri << 3 | fan triangle) per tile each fan triangle
// touches, in fan order; returns their number
template <bool kCull, typename Keep, typename Xf, typename F>
__device__ __forceinline__ uint32_t clip_visit(const float4* tris, uint32_t tri, uint32_t width, uint32_t height, Keep&& keep, Xf&& xf,
                                               F&& f) {
    if (!keep(tri)) return 0;
    float4 v[kClipMaxPoly];
    const int np = clip_tri_poly(tris, tri, xf, v);
    const int tx = tiles_x(width);
    uint32_t cnt = 0;
    for (int k = 0; k + 2 < np; ++k) {
        FanTri d;
        clip_fan<kCull>(v, k, width, height, d);
        cnt += tile_walk_tri(d.t, tx, [&](uint32_t, uint32_t tile) { f(tile, tri << 3 | (uint32_t)k); });
    }
    return cnt;
}

// ---- the tile kernels' fan triangles -------------------------------------------------------------------------------
struct FanEdges {
    int32_t A[3][kTileThreads], B[3][kTileThreads];
    long long C[3][kTileThreads];   // exact edge values at the tile's pixel (0, 0)
    float z[3][kTileThreads];
    uint32_t incl[kTileThreads];    // bit k: edge k owns the samples on it (top-left rule)
};

// stages fan triangle k of polygon v in slot `slot`, edge values relative to pixel (ox, oy)
template <bool kCull, typename V>
__device__ __forceinline__ void clip_stage(const V (&v)[kClipMaxPoly], int k, uint32_t width, uint32_t height, int ox, int oy,
                                           FanEdges& s, int slot) {
    FanTri d;
    clip_fan<kCull>(v, k, width, height, d);
    uint32_t incl = 0;
#pragma unroll
    for (int e = 0; e < 3; ++e) {
        s.A[e][slot] = d.t.A[e];
        s.B[e][slot] = d.t.B[e];
        s.C[e][slot] = d.t.C[e] + (long long)d.t.A[e] * ox + (long long)d.t.B[e] * oy;
        s.z[e][slot] = d.z[e];
        incl |= d.t.incl[e] ? 1u << e : 0u;
    }
    s.incl[slot] = incl;
}

// does staged fan triangle j cover pixel (lx, ly) of the tile, and with which D24 code?  GL 4.6 §14.6.1: z = ((E0 z0 +
// E1 z1) + E2 z2) / (E0 + E1 + E2), fp64 (the E are exact below 2^46); false outside or for a NaN depth (no write)
__device__ __forceinline__ bool clip_depth(const FanEdges& s, uint32_t j, int lx, int ly, uint32_t& code) {
    const uint32_t incl = s.incl[j];
    long long e[3];
    bool in = true;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        e[k] = s.C[k][j] + (long long)s.A[k][j] * lx + (long long)s.B[k][j] * ly;
        in &= e[k] >= ((incl >> k & 1u) ? 0ll : 1ll);
    }
    if (!in) return false;
    const double num = __dadd_rn(__dadd_rn(__dmul_rn((double)e[0], (double)s.z[0][j]), __dmul_rn((double)e[1], (double)s.z[1][j])),
                                 __dmul_rn((double)e[2], (double)s.z[2][j]));
    return d24_encode(__ddiv_rn(num, (double)(e[0] + e[1] + e[2])), code);
}

}  // namespace m2s
