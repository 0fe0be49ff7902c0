// m2s_gauss.cuh — what the two consumers of gaussian records share: the viewer prepass (m2s_prepass.cu) and the standard
// 3DGS render (m2s_3dgs.cu).  The fields of a record for each record layout, and the view-dependent colour from the SH
// rest coefficients of a loaded .ply (graphdeco's computeColorFromSH with its constants and the signs folded into the
// basis; every operation one round-to-nearest fp32 step without contraction, as oracle/m2s_sh_oracle.c restates it).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "m2s_tile.cuh"

namespace m2s {

// one gaussian as the prepass shader sees it (GaussianVertex): position, colour and alpha, scale, normal, rotation
// (w, x, y, z) and the two PBR values
struct GaussFields {
    float px, py, pz, cr, cg, cb, ca, sx, sy, sz, nx, ny, nz, qx, qy, qz, qw, pb0, pb1;
};

// REF96: position color scale normal rotation pbr, one float4 each
__device__ __forceinline__ void ref96_fields(const float4& p, const float4& c, const float4& s, const float4& nn, const float4& q,
                                             const float4& pb, GaussFields& g) {
    g.px = p.x; g.py = p.y; g.pz = p.z; g.cr = c.x; g.cg = c.y; g.cb = c.z; g.ca = c.w; g.sx = s.x; g.sy = s.y; g.sz = s.z;
    g.nx = nn.x; g.ny = nn.y; g.nz = nn.z; g.qx = q.x; g.qy = q.y; g.qz = q.z; g.qw = q.w; g.pb0 = pb.x; g.pb1 = pb.y;
}

// PACKED56: xyz | quat wxyz | log-scale | SH0 | opacity logit, seven float2 (parsers.cpp:560-622 on load): scale =
// exp(log-scale), colour = SH0 C0 + 0.5, alpha = 1 / (1 + exp(-logit)); no normal, no PBR values.  kExact: rn_exp and
// round-to-nearest steps without contraction (the 3DGS render, DESIGN §2); otherwise expf and the compiler's
// contraction, as the viewer prepass has always computed them.
template <bool kExact>
__device__ __forceinline__ void packed56_fields(const float2& f0, const float2& f1, const float2& f2, const float2& f3, const float2& f4,
                                                const float2& f5, const float2& f6, GaussFields& g) {
    g.px = f0.x; g.py = f0.y; g.pz = f1.x; g.qx = f1.y; g.qy = f2.x; g.qz = f2.y; g.qw = f3.x;
    const float kC0 = 0.28209479177387814f;
    if (kExact) {
        g.sx = rn_exp(f3.y); g.sy = rn_exp(f4.x); g.sz = rn_exp(f4.y);
        g.cr = ad(ml(f5.x, kC0), 0.5f); g.cg = ad(ml(f5.y, kC0), 0.5f); g.cb = ad(ml(f6.x, kC0), 0.5f);
        g.ca = dv(1.0f, ad(1.0f, rn_exp(-f6.y)));
    } else {
        g.sx = expf(f3.y); g.sy = expf(f4.x); g.sz = expf(f4.y);
        g.cr = f5.x * kC0 + 0.5f; g.cg = f5.y * kC0 + 0.5f; g.cb = f6.x * kC0 + 0.5f;
        g.ca = 1.0f / (1.0f + expf(-f6.y));
    }
    g.nx = g.ny = g.nz = 0.0f; g.pb0 = g.pb1 = 0.0f;
}

// ---- view-dependent colour (m2s_prepass_sh, m2s_3dgs_render) -----------------------------------------------------------
// rest = sum over k = 1..K of B_k coeff_k, in k order per channel; c: the gaussian's block (coefficient-major r g b)
template <int D>
__device__ __forceinline__ void sh_rest(const float4* c, float x, float y, float z, float rest[3]) {
    constexpr int K = (D + 1) * (D + 1) - 1;
    const float C1 = 0.4886025119029199f;
    float B[15];
    B[0] = __fmul_rn(-C1, y); B[1] = __fmul_rn(C1, z); B[2] = __fmul_rn(-C1, x);
    if (D >= 2) {
        const float xx = __fmul_rn(x, x), yy = __fmul_rn(y, y), zz = __fmul_rn(z, z);
        const float xy = __fmul_rn(x, y), yz = __fmul_rn(y, z), xz = __fmul_rn(x, z);
        B[3] = __fmul_rn(1.0925484305920792f, xy);
        B[4] = __fmul_rn(-1.0925484305920792f, yz);
        B[5] = __fmul_rn(0.31539156525252005f, __fsub_rn(__fsub_rn(__fmul_rn(2.0f, zz), xx), yy));
        B[6] = __fmul_rn(-1.0925484305920792f, xz);
        B[7] = __fmul_rn(0.5462742152960396f, __fsub_rn(xx, yy));
        if (D >= 3) {
            B[8] = __fmul_rn(__fmul_rn(-0.5900435899266435f, y), __fsub_rn(__fmul_rn(3.0f, xx), yy));
            B[9] = __fmul_rn(__fmul_rn(2.890611442640554f, xy), z);
            B[10] = __fmul_rn(__fmul_rn(-0.4570457994644658f, y), __fsub_rn(__fsub_rn(__fmul_rn(4.0f, zz), xx), yy));
            B[11] = __fmul_rn(__fmul_rn(0.3731763325901154f, z), __fsub_rn(__fsub_rn(__fmul_rn(2.0f, zz), __fmul_rn(3.0f, xx)), __fmul_rn(3.0f, yy)));
            B[12] = __fmul_rn(__fmul_rn(-0.4570457994644658f, x), __fsub_rn(__fsub_rn(__fmul_rn(4.0f, zz), xx), yy));
            B[13] = __fmul_rn(__fmul_rn(1.445305721320277f, z), __fsub_rn(xx, yy));
            B[14] = __fmul_rn(__fmul_rn(-0.5900435899266435f, x), __fsub_rn(xx, __fmul_rn(3.0f, yy)));
        }
    }
    rest[0] = rest[1] = rest[2] = 0.0f;
#pragma unroll
    for (int v = 0; v < (3 * K + 3) / 4; ++v) {   // every load of the block first: one round trip to memory
        const float4 q = __ldg(c + v);
        const float e[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (4 * v + j < 3 * K) rest[(4 * v + j) % 3] = __fadd_rn(rest[(4 * v + j) % 3], __fmul_rn(B[(4 * v + j) / 3], e[j]));
    }
}

// the colour of gaussian gid at model-space position p seen from cam (the camera in model space), degree 1..3 of the
// buffer sh (vec4 float4 per gaussian): max(colour + rest, 0) per channel (glm::max: NaN kept)
__device__ __forceinline__ void sh_colour(const float4* sh, uint32_t vec4, uint32_t degree, const float* cam, unsigned long long gid, float px,
                                          float py, float pz, float& r, float& g, float& b) {
    const float dx = __fsub_rn(px, cam[0]), dy = __fsub_rn(py, cam[1]), dz = __fsub_rn(pz, cam[2]);
    const float len = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
    float rest[3] = {0.0f, 0.0f, 0.0f};
    if (len != 0.0f) {
        const float inv = __fdiv_rn(1.0f, len);
        const float x = __fmul_rn(dx, inv), y = __fmul_rn(dy, inv), z = __fmul_rn(dz, inv);
        const float4* c = sh + gid * vec4;
        if (degree == 1) sh_rest<1>(c, x, y, z, rest);
        else if (degree == 2) sh_rest<2>(c, x, y, z, rest);
        else sh_rest<3>(c, x, y, z, rest);
    }
    r = __fadd_rn(r, rest[0]); g = __fadd_rn(g, rest[1]); b = __fadd_rn(b, rest[2]);
    r = r < 0.0f ? 0.0f : r; g = g < 0.0f ? 0.0f : g; b = b < 0.0f ? 0.0f : b;
}

}  // namespace m2s
