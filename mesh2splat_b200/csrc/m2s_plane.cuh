// m2s_plane.cuh — where a triangle lands on the pixel grid: its face frame and its dominant-axis orthographic uv
// (converterGS.glsl:327-397), as the raster kernel's set-up computes them (m2s_raster.cu), and the density bound derived
// from them when a scene is uploaded (m2s_scene.cu): one definition, so the bound is a bound of the set-up's own box.
#pragma once
#include "m2s_device.cuh"

namespace m2s {

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

// converterGS.glsl:327-397: the longest edge e1 (normalised), the face normal n, and the orthographic uv (ou, ov) of the
// three vertices over the primitive's box: X-dominant -> (y,z), Y -> (x,z), Z -> (x,y), over max(range_a, range_b).
// The rasterised plane is this uv plane scaled by R, not the mesh's own uv.
__device__ __forceinline__ void ortho_uv(const f3 (&P)[3], const DPrim& pr, f3& e1, f3& n, float (&ou)[3], float (&ov)[3]) {
    e1 = sub3(P[1], P[0]);
    f3 e2 = sub3(P[2], P[0]), e3 = sub3(P[2], P[1]);
    const float l1 = len3(e1), l2 = len3(e2), l3 = len3(e3);
    if (l2 > l1 && l2 > l3) { f3 tmp = e1; e1 = e2; e2 = tmp; }
    else if (l3 > l1 && l3 > l2) { e1 = e3; }
    e1 = norm3(e1);
    n = norm3(cross3(e1, e2));
    const float ax = fabsf(n.x), ay = fabsf(n.y), az = fabsf(n.z);
    const int axis = (ax > ay && ax > az) ? 0 : ((ay > az) ? 1 : 2);
    const float mina = axis == 0 ? pr.bmin[1] : pr.bmin[0], maxa = axis == 0 ? pr.bmax[1] : pr.bmax[0];
    const float minb = axis == 2 ? pr.bmin[1] : pr.bmin[2], maxb = axis == 2 ? pr.bmax[1] : pr.bmax[2];
    const float ra = __fsub_rn(maxa, mina), rb = __fsub_rn(maxb, minb);
    const float range = (ra < rb) ? rb : ra;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float pa = axis == 0 ? P[k].y : P[k].x, pb = axis == 2 ? P[k].y : P[k].z;
        ou[k] = __fdiv_rn(__fsub_rn(pa, mina), range);
        ov[k] = __fdiv_rn(__fsub_rn(pb, minb), range);
    }
}

// The largest density R at which the set-up's candidate box of a triangle whose orthographic uv spans eu x ev is
// certainly small (at most kSmallCand pixels and 32 rows); +inf for a triangle the set-up drops at every density.
// The box's width is at most floor(eu R + 1/64) + 1: the box counts the pixel centres between the snapped extremes, at
// most floor(D / 256) + 1 for a fixed-point extent D <= 256 (xw_max - xw_min) + 1, and xw_max - xw_min exceeds eu R by
// the roundings of xw = (2 ou - 1) R/2 + R/2 and of eu, under 0.005 pixels inside the guard band (|xw| <= kGuard).  So
// a w x h box needs eu R + 1/64 < w, which R <= (w - 1/32) / eu guarantees; the rows likewise.  The result is the best
// split of the 64 pixels into w columns and min(32, 64 / w) rows.  A small box also keeps the walk's edge functions
// int32-safe: every |E| inside it is below 4 * 65536 * 64.
__device__ __forceinline__ float small_box_density(float eu, float ev) {
    if (!(eu >= 0.0f) || !(ev >= 0.0f) || isinf(eu) || isinf(ev)) return INFINITY;   // not finite: never rasterised
    float best = 0.0f;
    for (uint32_t w = 1; w <= kSmallCand; ++w) {
        const float h = (float)min(32u, kSmallCand / w);
        const float rw = eu > 0.0f ? (w - 0.03125f) / eu : INFINITY;
        const float rh = ev > 0.0f ? (h - 0.03125f) / ev : INFINITY;
        best = fmaxf(best, fminf(rw, rh));
    }
    return best;
}

}  // namespace m2s
