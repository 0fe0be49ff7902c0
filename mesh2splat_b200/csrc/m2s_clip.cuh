// m2s_clip.cuh — the clip-space stage the mesh passes share: the mesh depth pre-pass (m2s_depth.cu) and the mesh G-buffer
// pass (m2s_mesh.cu).  GLM's mat4 * vec4, Sutherland-Hodgman against the six planes (z against +-w, x and y against a
// guard band of +-kDepthGuard w), the fan of the clipped polygon, the splat draw's viewport snap and edge set-up, and the
// walk over the 16 x 16 tiles a fan triangle touches (DESIGN §2).  Every operation is round-to-nearest fp32 with no
// contraction, so the oracles restate it bit for bit.
//
// The clipper is a template over the polygon vertex: a bare float4 (the depth pass) or a ClipVert, which carries each
// vertex's barycentric weights with respect to its source triangle through the cuts (the G-buffer pass interpolates its
// varyings from them).  Both clip the positions with the same operations, so their polygons are the same.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "m2s_depth.cuh"
#include "m2s_splat.cuh"

namespace m2s {

// GLM mat4 * vec4(x, y, z, w), column-major m: (m0 x + m1 y) + (m2 z + m3 w)
__device__ __forceinline__ float clip_row(const float* m, int row, float x, float y, float z, float w) {
    return __fadd_rn(__fadd_rn(__fmul_rn(m[row], x), __fmul_rn(m[4 + row], y)), __fadd_rn(__fmul_rn(m[8 + row], z), __fmul_rn(m[12 + row], w)));
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
    const float gw = __fmul_rn(kDepthGuard, v.w);
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
// vertex count (0: nothing left, or a coordinate of v[0..2] is not finite).  A polygon that would grow past kDepthMaxPoly
// vertices (only through rounding) keeps its first kDepthMaxPoly.
template <typename V>
__device__ int clip_poly(V (&v)[kDepthMaxPoly]) {
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
        V o[kDepthMaxPoly];
        int m = 0;
        float dp = clip_plane(clip_pos(v[n - 1]), p);
        for (int i = 0; i < n; ++i) {
            const float dc = clip_plane(clip_pos(v[i]), p);
            const int prev = i == 0 ? n - 1 : i - 1;
            if (dc >= 0.0f) {
                if (dp < 0.0f && m < kDepthMaxPoly) o[m++] = clip_cut(v[i], v[prev], dc, dp);
                if (m < kDepthMaxPoly) o[m++] = v[i];
            } else if (dp >= 0.0f && m < kDepthMaxPoly) {
                o[m++] = clip_cut(v[prev], v[i], dp, dc);
            }
            dp = dc;
        }
        for (int i = 0; i < m; ++i) v[i] = o[i];
        n = m;
    }
    return n;
}

struct DepthTri {
    SplatTri t;
    float z[3];   // window depth (z / w) 0.5 + 0.5 of the three vertices
};

// fan triangle (v0, vk+1, vk+2) of a W x H viewport: perspective divide, the splat draw's viewport transform, snap and
// edge set-up.  kCull: a triangle whose snapped window-space area is negative (clockwise, y up) is set up empty, as a
// zero area always is (GL_CULL_FACE with glCullFace(GL_BACK), glFrontFace(GL_CCW)).
template <bool kCull, typename V>
__device__ __forceinline__ void clip_fan(const V (&v)[kDepthMaxPoly], int k, uint32_t width, uint32_t height, DepthTri& d) {
    const float hw = __fmul_rn((float)width, 0.5f), hh = __fmul_rn((float)height, 0.5f);
    int X[3], Y[3];
    bool ok = true;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float4& p = clip_pos(v[c == 0 ? 0 : k + c]);
        bool okc;
        splat_snap(__fdiv_rn(p.x, p.w), __fdiv_rn(p.y, p.w), hw, hh, okc, X[c], Y[c]);
        ok &= okc;
        d.z[c] = __fadd_rn(__fmul_rn(__fdiv_rn(p.z, p.w), 0.5f), 0.5f);
    }
    if (kCull && ok) ok = (long long)(X[1] - X[0]) * (Y[2] - Y[0]) - (long long)(X[2] - X[0]) * (Y[1] - Y[0]) >= 0;
    splat_tri_setup(X, Y, ok, (int)width, (int)height, d.t);
}

__device__ __forceinline__ int clip_tiles_x(uint32_t width) { return (int)((width + kSplatTile - 1) / kSplatTile); }

// visits the tiles the fan triangle touches in tile-id order; returns their number
template <typename F>
__device__ __forceinline__ uint32_t clip_for_each_tile(const SplatTri& t, int tiles_x, F&& f) {
    if (t.x1 < t.x0 || t.y1 < t.y0) return 0;
    uint32_t c = 0;
    for (int ty = t.y0 / kSplatTile; ty <= t.y1 / kSplatTile; ++ty)
        for (int tx = t.x0 / kSplatTile; tx <= t.x1 / kSplatTile; ++tx)
            if (splat_tri_touches(t, tx, ty)) f(c++, (uint32_t)(ty * tiles_x + tx));
    return c;
}

}  // namespace m2s
